"""Free-space kernels (csrc/freespace.cu) against the C oracle, bit for bit: crop box, labels, both count arrays and the .grid
bytes, over frame sizes, seeds, noise, dropped pixels, frames without a pose, camera paths that put many bricks on the frustum
border, batchings, the .sens scene driver and the CLI."""
import os
import subprocess
import zlib

import numpy as np
import pytest

import freespace_bindings as fb
from scannet_b200 import ScnError, synth
from scannet_b200 import freespace as fsp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(g, o):
    glo, gd, gl, gf, gn = g
    olo, od, ol, of, on = o
    assert tuple(glo) == tuple(olo) and tuple(gd) == tuple(od), (glo, gd, olo, od)
    assert gl.tobytes() == ol.tobytes() and gf.tobytes() == of.tobytes() and gn.tobytes() == on.tobytes()


def _gpu(p, lo, dims, W, H, D, P, K, splits=None):
    with fsp.FreeSpace(lo, dims, W, H, params=p) as h:
        if splits is None:
            h.integrate(D, P, K)
        else:
            i = 0
            while i < len(P):
                h.integrate(D[i:i + splits], P[i:i + splits], K)
                i += splits
        return h.download(), h.report()


def _frames(W, H, n, seed, noise_mm=0.0, drop=0.0, invalid_pose_every=0, loop=None):
    D, _, P, K = synth.make_frames(n, seed=seed, width=W, height=H, noise_mm=noise_mm, drop=drop, invalid_pose_every=invalid_pose_every,
                                   loop_frames=loop or n, with_color=False)
    return D, P, K


@pytest.mark.parametrize("W,H,n,seed,noise,drop,vs", [(640, 480, 12, 0, 0.0, 0.0, 0.05), (640, 480, 10, 4, 3.0, 0.05, 0.05),
                                                      (96, 72, 40, 1, 2.0, 0.02, 0.05), (161, 119, 33, 2, 1.0, 0.1, 0.04),
                                                      (161, 119, 20, 3, 0.0, 0.0, 0.1)])
def test_kernels_equal_oracle(built, tmp_path, W, H, n, seed, noise, drop, vs):
    D, P, K = _frames(W, H, n, seed, noise, drop, invalid_pose_every=7, loop=60)
    p = fsp.default_params(voxel_size=vs, band_base=vs)
    lo, dims = fsp.envelope(P, K, W, H, p)
    g, rep = _gpu(p, lo, dims, W, H, D, P, K)
    o = fb.oracle_grid(p, lo, dims, W, H, D, P, K)
    _same(g, o)
    assert rep["frames_used"] == n - n // 7 and rep["frames_skipped_pose"] == n // 7
    assert rep["voxels_free"] == (o[2] == 1).sum() and rep["voxels_occupied"] == (o[2] == 2).sum()
    assert rep["voxels_unknown"] == (o[2] == 0).sum() and rep["voxels_occupied"] > 0
    assert 0 < rep["pairs_classified"] < rep["pairs_classified"] + rep["pairs_culled"]
    path = tmp_path / "g.grid"
    fsp.save_grid(path, p.voxel_size, g[0], g[1], g[2])
    assert path.read_bytes() == fb.grid_bytes(np.float32(vs), o[0], o[1], o[2])


def test_frustum_border_camera_path(built):
    """Cameras at random positions and orientations, an odd voxel size and an envelope offset from the brick lattice, so that
    many bricks straddle a frustum plane, the near plane or the far limit."""
    W, H = 161, 119
    rng = np.random.default_rng(11)
    sc = synth.BoxRoomScene(seed=6, width=W, height=H, fx=synth.FX * W / 640, fy=synth.FY * H / 480, cx=(W - 1) / 2, cy=(H - 1) / 2)
    P = []
    for _ in range(24):
        a, b, c = rng.uniform(-np.pi, np.pi, 3)
        Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
        Rx = np.array([[1, 0, 0], [0, np.cos(c), -np.sin(c)], [0, np.sin(c), np.cos(c)]])
        T = np.eye(4); T[:3, :3] = Rz @ Ry @ Rx; T[:3, 3] = rng.uniform([0.5, 0.5, 0.3], np.asarray(sc.size) - 0.5)
        P.append(T.astype(np.float32))
    P = np.stack(P)
    D = np.stack([sc.render(P[i], noise_mm=1.0, frame_seed=i)[0] for i in range(len(P))])
    K = sc.intrinsics()
    p = fsp.default_params(voxel_size=0.037, band_base=0.03, max_distance=3.3)
    lo, dims = fsp.envelope(P, K, W, H, p)
    lo = lo - np.array([3, 5, 1], np.int32); dims = dims + np.array([6, 3, 9], np.uint64)
    g, rep = _gpu(p, lo, dims, W, H, D, P, K)
    _same(g, fb.oracle_grid(p, lo, dims, W, H, D, P, K))
    assert rep["pairs_culled"] > rep["pairs_classified"] > 0


def test_batching_invariance(built):
    W, H = 96, 72
    D, P, K = _frames(W, H, 70, 5, 2.0, 0.03, invalid_pose_every=9, loop=70)
    p = fsp.default_params()
    lo, dims = fsp.envelope(P, K, W, H, p)
    whole, rep = _gpu(p, lo, dims, W, H, D, P, K)
    _same(whole, fb.oracle_grid(p, lo, dims, W, H, D, P, K))
    for s in (1, 7, 32, 33):
        g, r = _gpu(p, lo, dims, W, H, D, P, K, splits=s)
        _same(g, whole)
        assert r["pairs_classified"] == rep["pairs_classified"] and r["frames_used"] == rep["frames_used"]


def _write_sens(path, D, P, K, corrupt=()):
    """zlib depth, no colour; frames in `corrupt` get a depth payload that does not inflate"""
    N, H, W = D.shape
    with synth.SensWriter(path, N, (W, H), (0, 0), K, color_comp=0) as wr:
        for i in range(N):
            wr.add(b"", b"\x00garbage" * 9 if i in corrupt else zlib.compress(D[i].tobytes(), 6), P[i])


def test_scene_driver_equals_host_frames_and_oracle(built, tmp_path):
    W, H = 161, 119
    D, P, K = _frames(W, H, 45, 8, 2.0, 0.02, loop=45)
    P[[3, 17, 30]] = -np.inf
    sens = str(tmp_path / "scene.sens")
    _write_sens(sens, D, P, K, corrupt={17})                        # a pose-less frame whose payload is corrupt is never decoded
    p = fsp.default_params()
    out = tmp_path / "scene.grid"
    rep = fsp.freespace_scene(sens, out, p)
    assert rep["frames_used"] == 42 and rep["frames_skipped_pose"] == 3
    lo, dims = fsp.envelope(P, K, W, H, p)
    assert list(lo) == rep["envelope_lo"] and list(dims) == rep["envelope_dims"]
    host, hrep = _gpu(p, lo, dims, W, H, D, P, K)
    o = fb.oracle_grid(p, lo, dims, W, H, D, P, K)
    _same(host, o)
    assert out.read_bytes() == fb.grid_bytes(np.float32(p.voxel_size), o[0], o[1], o[2])
    assert rep["pairs_classified"] == hrep["pairs_classified"] and rep["output_dims"] == list(o[1])
    g = fsp.read_grid(out)
    assert (g["labels"] == o[2]).all()


def test_scene_driver_raw_depth(built, tmp_path):
    """uncompressed depth payloads go through the driver's upload branch; same grid as the zlib file and the oracle"""
    W, H = 96, 72
    D, P, K = _frames(W, H, 20, 12, 1.0, 0.02, invalid_pose_every=6, loop=20)
    raw, zl = str(tmp_path / "raw.sens"), str(tmp_path / "zlib.sens")
    synth.write_sens(raw, D, None, P, K, depth_comp=0)
    _write_sens(zl, D, P, K)
    p = fsp.default_params()
    before = bytes(p)
    r1 = fsp.freespace_scene(raw, tmp_path / "raw.grid", p, voxel_size=0.08, band_base=0.08)
    assert bytes(p) == before, "keyword overrides must not write into the caller's params"
    r2 = fsp.freespace_scene(zl, tmp_path / "zlib.grid", p, voxel_size=0.08, band_base=0.08)
    assert (tmp_path / "raw.grid").read_bytes() == (tmp_path / "zlib.grid").read_bytes()
    assert r1["frames_used"] == r2["frames_used"] == 17
    p2 = fsp.default_params(voxel_size=0.08, band_base=0.08)
    lo, dims = fsp.envelope(P, K, W, H, p2)
    o = fb.oracle_grid(p2, lo, dims, W, H, D, P, K)
    assert (tmp_path / "raw.grid").read_bytes() == fb.grid_bytes(np.float32(0.08), o[0], o[1], o[2])


def test_scan_without_pose_gives_an_empty_grid(built, tmp_path):
    D, P, K = _frames(64, 48, 4, 1)
    P[:] = -np.inf
    sens = str(tmp_path / "none.sens")
    _write_sens(sens, D, P, K, corrupt={0, 2})
    rep = fsp.freespace_scene(sens, tmp_path / "none.grid")
    assert rep["frames_used"] == 0 and rep["frames_skipped_pose"] == 4 and rep["output_dims"] == [0, 0, 0]
    assert (tmp_path / "none.grid").read_bytes() == fb.grid_bytes(np.float32(0.05), (0, 0, 0), (0, 0, 0), np.zeros(0, np.uint8))


def test_corrupt_payload_of_a_posed_frame_fails(built, tmp_path):
    D, P, K = _frames(64, 48, 4, 1)
    sens = str(tmp_path / "bad.sens")
    _write_sens(sens, D, P, K, corrupt={2})
    with pytest.raises(ScnError):
        fsp.freespace_scene(sens, tmp_path / "bad.grid")


def test_capacity_refusal(built, tmp_path):
    D, P, K = _frames(64, 48, 3, 1)
    sens = str(tmp_path / "c.sens")
    _write_sens(sens, D, P, K)
    with pytest.raises(ScnError) as e:
        fsp.freespace_scene(sens, tmp_path / "c.grid", voxel_size=0.01, band_base=0.01, max_voxels=1 << 24)
    assert e.value.code == -5 and "exceeds max_voxels" in str(e.value)
    assert not (tmp_path / "c.grid").exists()


def test_cli(built, tmp_path):
    W, H = 96, 72
    D, P, K = _frames(W, H, 30, 9, 1.0, 0.0, invalid_pose_every=5, loop=30)
    sens = str(tmp_path / "scene0000_00.sens")
    _write_sens(sens, D, P, K)
    exe = os.path.join(ROOT, "scannet_b200/bin/freespace")
    r = subprocess.run([exe, sens], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    p = fsp.default_params()
    lo, dims = fsp.envelope(P, K, W, H, p)
    o = fb.oracle_grid(p, lo, dims, W, H, D, P, K)
    assert (tmp_path / "scene0000_00.grid").read_bytes() == fb.grid_bytes(np.float32(p.voxel_size), o[0], o[1], o[2])
    # a parameter file (depth range, max distance), an output path and --voxel
    prm = tmp_path / "params.txt"
    prm.write_text("s_sensorDepthMin = 0.2;\ns_sensorDepthMax = 5.0;\ns_SDFMaxIntegrationDistance = 3.0f;\ns_SDFVoxelSize = 0.9;\n")
    out = tmp_path / "other.grid"
    r = subprocess.run([exe, str(prm), sens, str(out), "--voxel", "0.08"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    p2 = fsp.default_params(depth_min=0.2, depth_max=5.0, max_distance=3.0, voxel_size=0.08, band_base=0.08)
    lo, dims = fsp.envelope(P, K, W, H, p2)
    o = fb.oracle_grid(p2, lo, dims, W, H, D, P, K)
    assert out.read_bytes() == fb.grid_bytes(np.float32(0.08), o[0], o[1], o[2])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 255 and "Usage" in r.stdout
