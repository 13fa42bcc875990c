"""Free-space spec v1 (DESIGN.md §6h) on the CPU: the C oracle against an independent float64 statement and against the analytic
box room, envelope invariance, the .grid format, the parameter refusals, and the library's behaviour without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import freespace_bindings as fb
import freespace_reference as fr
from scannet_b200 import ScnError, synth
from scannet_b200 import freespace as fsp
from scannet_b200._lib import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _room(W, H, n, seed=0, noise_mm=0.0, drop=0.0, loop=None):
    sc = synth.BoxRoomScene(seed=seed, width=W, height=H, fx=synth.FX * W / 640, fy=synth.FY * H / 480, cx=(W - 1) / 2, cy=(H - 1) / 2)
    P = np.stack([sc.camera_pose(i, loop or n) for i in range(n)])
    D = np.stack([sc.render(P[i], noise_mm=noise_mm, drop=drop, frame_seed=i)[0] for i in range(n)])
    return sc, D, P, sc.intrinsics()


@pytest.mark.parametrize("W,H,vs,seed", [(96, 72, 0.1, 3), (161, 119, 0.05, 5)])
def test_oracle_matches_float64_statement(built, W, H, vs, seed):
    """Labels and counts identical on every voxel whose deciding quantities all lie more than eps (1e-4 m, 2e-3 px) from a
    threshold in every frame; the excluded voxels are counted (a few tenths of a percent of the box)."""
    _, D, P, K = _room(W, H, 4, seed=seed, noise_mm=2.0, drop=0.02, loop=24)
    p = fsp.default_params(voxel_size=vs, band_base=vs)
    lo, dims = fsp.envelope(P, K, W, H, p)
    o = fb.OracleCounts(p, lo, dims, W, H).integrate(D, P, K)
    nf, no, amb = fr.counts_f64(p, lo, dims, W, H, D, P, K)
    keep = ~amb
    lab_o, lab_r = fb.labels_of(o.n_free, o.n_occ), fb.labels_of(nf, no)
    print(f"{W}x{H} vs={vs}: {amb.sum()} of {amb.size} voxels excluded, {(lab_o > 0).sum()} labelled")
    assert amb.sum() < 0.01 * amb.size
    assert (lab_o > 0).sum() > 1000
    assert (lab_o[keep] == lab_r[keep]).all()
    assert (o.n_free[keep] == nf[keep]).all() and (o.n_occ[keep] == no[keep]).all()


def test_box_room_geometry(built):
    """24 noiseless 160x120 frames of one camera loop at 5 cm.  Margins calibrated on the oracle: band(6 m) = 0.11 m plus one
    voxel and a little; 94 % of the observed voxels within one voxel of a surface are occupied."""
    W, H = 160, 120
    sc, D, P, K = _room(W, H, 24)
    p = fsp.default_params()
    lo, dims = fsp.envelope(P, K, W, H, p)
    o = fb.OracleCounts(p, lo, dims, W, H).integrate(D, P, K)
    lab = fb.labels_of(o.n_free, o.n_occ)
    gz, gy, gx = np.meshgrid(*(np.arange(int(dims[a])) + lo[a] for a in (2, 1, 0)), indexing="ij")
    X = np.stack([gx, gy, gz], -1) * p.voxel_size
    S = np.asarray(sc.size)
    d_room = np.min(np.concatenate([X, S - X], -1), -1)                                     # > 0 inside the room
    d_sph = np.min(np.stack([np.linalg.norm(X - c, axis=-1) - r for c, r in sc.spheres], -1), -1)   # > 0 outside every sphere
    assert (lab[d_room < -0.15] == 0).all(), "voxels well outside the room must be unknown"
    interior = (d_room > 0.15) & (d_sph > 0.15)
    assert (lab[interior] != 2).all(), "voxels away from every surface must never be occupied"
    assert (lab[interior] == 1).sum() > 100000
    surf = np.minimum(np.abs(d_room), np.where(d_room > -p.voxel_size, np.abs(d_sph), np.inf)) <= p.voxel_size
    seen = surf & (lab > 0)
    assert seen.sum() > 10000
    assert ((lab == 2) & surf).sum() >= 0.9 * seen.sum()


def test_envelope_covers_and_a_larger_one_changes_nothing(built):
    W, H = 96, 72
    _, D, P, K = _room(W, H, 5, seed=1, noise_mm=1.0, loop=20)
    p = fsp.default_params(voxel_size=0.1, band_base=0.1)
    lo, dims = fsp.envelope(P, K, W, H, p)
    a = fb.oracle_grid(p, lo, dims, W, H, D, P, K)
    lo2 = lo - np.array([3, 7, 2], np.int32); dims2 = dims + np.array([9, 8, 11], np.uint64)
    b = fb.oracle_grid(p, lo2, dims2, W, H, D, P, K)
    assert (a[0] == b[0]).all() and a[1] == b[1]
    for x, y in zip(a[2:], b[2:]):
        assert x.tobytes() == y.tobytes()
    # the box is strictly inside the envelope: nothing is observed at its faces
    assert all(a[0][i] > lo[i] and a[0][i] + a[1][i] < lo[i] + int(dims[i]) for i in range(3))


def test_envelope_skips_invalid_poses_and_is_empty_without_any(built):
    _, _, P, K = _room(64, 48, 4, loop=8)
    p = fsp.default_params()
    lo, dims = fsp.envelope(P, K, 64, 48, p)
    P2 = P.copy(); P2[1] = -np.inf
    P2[1, 0, 3] = 1e9                       # a frame without pose carries no usable translation
    lo2, dims2 = fsp.envelope(P2, K, 64, 48, p)
    lo3, dims3 = fsp.envelope(P[[0, 2, 3]], K, 64, 48, p)
    assert (lo2 == lo3).all() and (dims2 == dims3).all()
    assert (lo2 >= lo).all()
    lo4, dims4 = fsp.envelope(np.full((3, 4, 4), -np.inf, np.float32), K, 64, 48, p)
    assert (dims4 == 0).all() and (lo4 == 0).all()


def test_grid_round_trip(built, tmp_path):
    rng = np.random.default_rng(0)
    lab = rng.integers(0, 3, (5, 4, 7)).astype(np.uint8)
    lo, dims = np.array([-3, 12, -40], np.int32), (7, 4, 5)
    path = tmp_path / "a.grid"
    fsp.save_grid(path, 0.05, lo, dims, lab)
    assert path.read_bytes() == fb.grid_bytes(np.float32(0.05), lo, dims, lab)
    g = fsp.read_grid(path)
    assert g["dims"] == dims and g["lo"] == tuple(lo) and (g["labels"] == lab).all() and g["voxel_size"] == np.float32(0.05)
    assert np.allclose(g["grid2world"] @ [1, 2, 3, 1], [(1 - 3) * g["voxel_size"], (2 + 12) * g["voxel_size"], (3 - 40) * g["voxel_size"], 1])
    empty = tmp_path / "e.grid"
    fsp.save_grid(empty, 0.05, np.zeros(3, np.int32), (0, 0, 0), np.zeros(0, np.uint8))
    assert empty.read_bytes() == fb.grid_bytes(np.float32(0.05), (0, 0, 0), (0, 0, 0), np.zeros(0, np.uint8))
    assert fsp.read_grid(empty)["labels"].size == 0


@pytest.mark.parametrize("field,value", [("voxel_size", 0.0), ("voxel_size", -0.1), ("voxel_size", float("nan")),
                                         ("band_base", -0.01), ("band_scale", float("nan")), ("depth_min", 6.0),
                                         ("max_distance", 0.0), ("max_distance", float("nan"))])
def test_parameter_refusals(built, field, value):
    p = fsp.default_params(**{field: value})
    K = np.eye(4, dtype=np.float32); K[0, 0] = K[1, 1] = 100
    with pytest.raises(ScnError) as e:
        fsp.envelope(np.eye(4, dtype=np.float32)[None], K, 64, 48, p)
    assert e.value.code == -1
    with pytest.raises(ScnError) as e:
        fsp.FreeSpace([0, 0, 0], [8, 8, 8], 64, 48, params=p)
    assert e.value.code == -1


def test_capacity_refusal_names_the_size(built):
    p = fsp.default_params(max_voxels=1000)
    with pytest.raises(ScnError) as e:
        fsp.FreeSpace([0, 0, 0], [10, 10, 11], 64, 48, params=p)
    assert e.value.code == -5 and "1100 voxels" in str(e.value)


def test_no_gpu_means_loud_failure(built, tmp_path):
    if lib().scn_device_count() > 0:
        return                      # on the GPU machine this test has nothing to show
    with pytest.raises(ScnError) as e:
        fsp.FreeSpace([0, 0, 0], [8, 8, 8], 64, 48)
    assert e.value.code == -2
    D, _, P, K = synth.make_frames(2, width=64, height=48, with_color=False)
    sens = tmp_path / "s.sens"
    synth.write_sens(str(sens), D, None, P, K)
    with pytest.raises(ScnError) as e:
        fsp.freespace_scene(sens, tmp_path / "s.grid")
    assert e.value.code == -2 and not (tmp_path / "s.grid").exists()


def test_report_binding_matches_the_library_struct(built):
    assert fsp.report_sizeof() == C.sizeof(fsp.FreespaceReport)


def test_cli_usage(built):
    r = subprocess.run([os.path.join(ROOT, "scannet_b200/bin/freespace")], capture_output=True, text=True)
    assert r.returncode == 255 and "Usage: freespace" in r.stdout
