"""GPU parity: mesh cleaning (scannet_b200/csrc/meshclean.cu through the C ABI) vs the CPU oracle (oracle/meshclean_oracle.c),
bit for bit: vertex bytes, colours, indices and every counter of the report."""
import json
import os
import subprocess

import numpy as np
import pytest

import meshclean_bindings as mb
import oracle_bindings as ob
from scannet_b200 import ScnError, meshclean, synth, tsdf

pytestmark = pytest.mark.gpu
ROOT = mb.ROOT
BIN = os.path.join(ROOT, "scannet_b200", "bin")
GOLDEN = os.path.join(ROOT, "tests", "golden")


def check(xyz, tri, rgb=None, **kw):
    gx, gc, gt, rep = meshclean.clean(xyz, tri, rgb, **kw)
    ox, oc, ot, cnt = mb.oracle_clean(xyz, tri, rgb, **kw)
    assert gx.tobytes() == ox.tobytes(), "vertices differ"
    assert (gc is None and oc is None) or gc.tobytes() == oc.tobytes(), "colours differ"
    assert gt.tobytes() == ot.tobytes(), "faces differ"
    assert {k: rep[k] for k in mb.COUNTERS} == cnt
    assert (rep["vertices_in"], rep["faces_in"], rep["vertices_out"], rep["faces_out"]) == (len(xyz), len(tri), len(ox), len(ot))
    return gx, gc, gt, rep


@pytest.fixture(scope="module")
def mc_mesh():
    """marching-cubes output of a fused synthetic scene at 4 mm voxels"""
    p = tsdf.default_params(width=160, height=120, voxel_size=0.004, max_blocks=1 << 16, hash_slots=1 << 18, batch_frames=4)
    D, C, P, K = synth.make_frames(8, seed=11, width=160, height=120, loop_frames=300, noise_mm=1.0)
    vol = tsdf.TsdfVolume(p, device=0)
    vol.integrate_batch(D, C, P, K)
    vol.sync()
    return vol.extract_mesh()


def test_gates381(built):
    xyz, rgb, tri = meshclean.load_rgb(os.path.join(GOLDEN, "gates381.ply"))
    _, _, _, rep = check(xyz, tri, rgb)                                    # clean.mlx: 4 duplicate faces, 9 of 10 pieces removed
    assert rep["duplicate_faces"] == 4 and rep["pieces_removed"] == 9
    for t, mf in ((0.03, 50), (0.05, 0), (0.05, 7500)):
        _, _, _, rep = check(xyz, tri, rgb, min_piece_faces=mf, merge_threshold=t)
        assert rep["vertices_merged"] > 0


@pytest.mark.parametrize("t", [0.0010689, 0.001, 0.002, 0.004])
def test_marching_cubes_mesh(built, mc_mesh, t):
    xyz, rgb, tri = mc_mesh
    assert len(tri) > 20000
    _, _, _, rep = check(xyz, tri, rgb, merge_threshold=t)
    assert rep["vertices_merged"] > 0
    print(f"t={t}: {rep['vertices_in']} -> {rep['vertices_out']} vertices, {rep['faces_in']} -> {rep['faces_out']} faces, "
          f"{rep['merge_components']} merge components (largest {rep['largest_merge_component']}), "
          f"merge {rep['merge_ms']:.2f} dedup {rep['dedup_ms']:.2f} pieces {rep['pieces_ms']:.2f} ms")


@pytest.mark.parametrize("flags", [mb.SKIP_DEDUP | mb.SKIP_PIECES, mb.SKIP_MERGE | mb.SKIP_PIECES, mb.SKIP_MERGE | mb.SKIP_DEDUP,
                                   mb.SKIP_MERGE | mb.SKIP_DEDUP | mb.SKIP_PIECES])
def test_each_step_alone(built, mc_mesh, flags):
    xyz, rgb, tri = mc_mesh
    tri = np.vstack([tri, tri[::7, ::-1], tri[::5]])                     # flipped and plain duplicates for the dedup step
    check(xyz, tri, rgb, flags=flags, merge_threshold=0.002, min_piece_faces=100, min_piece_vertices=60)


def test_piece_thresholds_and_noisy_fragments(built, mc_mesh):
    xyz, rgb, tri = mc_mesh
    rng = np.random.default_rng(5)
    frag = rng.uniform(0, 5, (3000, 3)).astype(np.float32)                # floating fragments: tiny disconnected triangles
    ftri = (np.arange(3000, dtype=np.uint32).reshape(-1, 3) + len(xyz))
    x = np.vstack([xyz, frag]); c = np.vstack([rgb, rng.integers(0, 256, (3000, 3)).astype(np.uint8)]); t = np.vstack([tri, ftri])
    for mv, mf in ((0, 0), (3, 1), (4, 0), (0, 2), (100, 7500)):
        _, _, _, rep = check(x, t, c, min_piece_vertices=mv, min_piece_faces=mf)
        if mv == 4 or mf == 2:
            assert rep["pieces_removed"] >= 1000


def test_adversarial_chain_is_one_component(built):
    """10^5 vertices 0.9 t apart on a line: one merge component; the rule alternates representative / merged"""
    n, t = 100000, np.float32(0.001)
    xyz = np.zeros((n, 3), np.float32)
    xyz[:, 0] = np.arange(n, dtype=np.float32) * np.float32(0.9) * t
    xyz[:, 1] = np.float32(0.25)
    tri = np.stack([np.arange(n - 2), np.arange(1, n - 1), np.arange(2, n)], 1).astype(np.uint32)
    gx, _, gt, rep = check(xyz, tri, None, merge_threshold=t, min_piece_faces=0)
    assert rep["merge_components"] == 1 and rep["largest_merge_component"] == n and rep["vertices_merged"] == n // 2
    print(f"chain of {n}: merge {rep['merge_ms']:.1f} ms, total {rep['total_ms']:.1f} ms")
    # the same chain in reverse order and a dense blob of identical points
    check(xyz[::-1].copy(), tri, None, merge_threshold=t, min_piece_faces=0)
    blob = np.repeat(np.array([[1.0, 2.0, 3.0]], np.float32), 5000, 0)
    _, _, _, r2 = check(blob, tri[:100], None, merge_threshold=t, min_piece_faces=0)
    assert r2["vertices_merged"] == 4999


def test_empty_and_faceless_and_everything_removed(built, mc_mesh):
    check(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint32))
    check(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint32), flags=mb.SKIP_MERGE)
    rng = np.random.default_rng(1)
    pts = rng.uniform(-1, 1, (5000, 3)).astype(np.float32)
    _, _, _, rep = check(pts, np.zeros((0, 3), np.uint32), None, merge_threshold=0.05)
    assert rep["vertices_out"] == 0
    check(pts, np.zeros((0, 3), np.uint32), None, merge_threshold=0.05, flags=mb.SKIP_PIECES)
    xyz, rgb, tri = mc_mesh
    _, _, gt, rep = check(xyz, tri, rgb, min_piece_faces=len(tri) + 1)
    assert len(gt) == 0 and rep["vertices_out"] == 0


def test_two_runs_identical(built, mc_mesh):
    xyz, rgb, tri = mc_mesh
    a = meshclean.clean(xyz, tri, rgb, merge_threshold=0.003)
    b = meshclean.clean(xyz, tri, rgb, merge_threshold=0.003)
    for u, v in zip(a[:3], b[:3]):
        assert u.tobytes() == v.tobytes()
    assert {k: a[3][k] for k in mb.COUNTERS} == {k: b[3][k] for k in mb.COUNTERS}


def test_refusals(built):
    xyz = np.zeros((3, 3), np.float32); tri = np.array([[0, 1, 2]], np.uint32)
    for t in (0.0, -0.001, float("nan")):
        with pytest.raises(ScnError) as e:
            meshclean.clean(xyz, tri, merge_threshold=t)
        assert e.value.code == -1
    for bad in (np.inf, -np.inf, np.nan, 3e6):
        x = xyz.copy(); x[2, 0] = bad
        with pytest.raises(ScnError) as e:
            meshclean.clean(x, tri, merge_threshold=0.001)
        assert e.value.code == -1
    with pytest.raises(ScnError) as e:
        meshclean.clean(xyz, np.array([[0, 1, 3]], np.uint32))
    assert e.value.code == -1
    x = xyz.copy(); x[2, 0] = np.inf                                       # merge skipped: coordinates are not looked at
    check(x, tri, None, flags=mb.SKIP_MERGE, merge_threshold=0.0, min_piece_faces=0)


def test_fuse_meshclean_segmentator_end_to_end(built, tmp_path):
    """synthetic .sens -> fuse -> _vh.ply -> meshclean (clean.mlx) -> _vh_clean.ply -> segmentator"""
    D, Cc, P, K = synth.make_frames(16, seed=4, width=160, height=120, loop_frames=600, noise_mm=1.5)
    sens = tmp_path / "scene.sens"
    synth.write_sens(str(sens), D, Cc, P, K, depth_comp=1, color_comp=0)
    params = tmp_path / "params.txt"
    params.write_text("s_SDFVoxelSize = 0.004f;\ns_SDFTruncation = 0.02f;\ns_SDFTruncationScale = 0.01f;\ns_hashNumSDFBlocks = 200000;\n")
    r = subprocess.run([os.path.join(BIN, "fuse"), str(params), str(sens)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    vh, clean = tmp_path / "scene_vh.ply", tmp_path / "scene_vh_clean.ply"
    r = subprocess.run([os.path.join(BIN, "meshclean"), "-i", str(vh), "-o", str(clean), "-m", "vc", "-s", os.path.join(GOLDEN, "clean.mlx")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "Merge Close Vertices" in r.stdout and "Remove Duplicate Faces" in r.stdout and "Remove Isolated pieces" in r.stdout
    xyz, rgb, tri = meshclean.load_rgb(str(vh))
    ox, oc, ot, _ = mb.oracle_clean(xyz, tri, rgb)
    assert len(ot) > 0
    want = tmp_path / "want.ply"
    from scannet_b200._lib import check as scn_check, lib
    import ctypes as C
    scn_check(lib().scn_mesh_save_ply(str(want).encode(), ox.ctypes.data_as(C.c_void_p), oc.ctypes.data_as(C.c_void_p), C.c_uint64(len(ox)),
                                      ot.ctypes.data_as(C.c_void_p), C.c_uint64(len(ot))))
    assert clean.read_bytes() == want.read_bytes()
    r = subprocess.run([os.path.join(BIN, "segmentator"), str(clean)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    seg = np.array(json.loads((tmp_path / "scene_vh_clean.0.010000.segs.json").read_text())["segIndices"])
    assert len(seg) == len(ox)
    assert (seg == ob.oracle_segment(ox, ot)).all()
    # the CLI without a script uses the clean.mlx defaults; without -m vc the colour is dropped (white)
    r = subprocess.run([os.path.join(BIN, "meshclean"), "-i", str(vh), "-o", str(tmp_path / "b.ply")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    bx, bc, bt = meshclean.load_rgb(str(tmp_path / "b.ply"))
    assert bx.tobytes() == ox.tobytes() and bt.tobytes() == ot.tobytes() and (bc == 255).all()
    r = subprocess.run([os.path.join(BIN, "meshclean"), "-i", str(vh), "-o", str(tmp_path / "c.ply"), "-s", os.path.join(GOLDEN, "simplify.mlx")],
                       capture_output=True, text=True)
    assert r.returncode != 0 and "Quadric Edge Collapse Decimation" in r.stderr
