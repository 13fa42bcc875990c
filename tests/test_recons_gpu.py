"""GPU tracker (csrc/track.cu) against the CPU oracle (oracle/track_oracle.c), bit for bit: per-frame poses, iterations, pair
counts, residual bits and lost flags, the final volume and its marching-cubes mesh; and the tracker's refusals."""
import os

import numpy as np
import pytest

import recons_bindings as rb
from scannet_b200 import ScnError, recons, synth, tsdf

pytestmark = pytest.mark.gpu


def scene(W, H, seed):
    return synth.BoxRoomScene(size=(5.0, 4.0, 3.0), n_spheres=10, seed=seed, width=W, height=H, fx=synth.FX * W / 640, fy=synth.FY * H / 480,
                              cx=(W - 1) / 2, cy=(H - 1) / 2)


def frames(sc, n, noise, drop, zero_at=None):
    D = np.zeros((n, sc.H, sc.W), np.uint16); C = np.zeros((n, sc.H, sc.W, 3), np.uint8); P = np.zeros((n, 4, 4), np.float32)
    for i in range(n):
        P[i] = sc.orbit_pose(i, 300, height=2.2)
        D[i], C[i] = sc.render(P[i], noise_mm=noise, drop=drop, frame_seed=i)
        if i == zero_at:
            D[i] = 0
    return D, C, P


def volume_params(W, H, depth_filter, max_blocks=1 << 15):
    return tsdf.default_params(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02, max_integration_distance=4.0, width=W, height=H,
                               max_blocks=max_blocks, hash_slots=1 << 17, batch_frames=1, depth_filter=depth_filter, depth_sigma_d=2.0,
                               depth_sigma_r=0.05)


CASES = [  # depth size, tracking size, filter, frames, noise mm, dropouts, seed, zero-depth frame
    ((320, 240), (320, 240), 1, 64, 1.0, 0.02, 2, 30),
    ((640, 480), (320, 240), 1, 60, 1.0, 0.0, 4, None),
    ((320, 240), (160, 120), 0, 64, 0.5, 0.02, 5, 40),
]


@pytest.mark.parametrize("case", CASES, ids=["320-filter-lost", "640to320-filter", "320to160-raw-lost"])
def test_tracker_bit_identical_to_oracle(built, case):
    (W, H), (tw, th), filt, n, noise, drop, seed, zero_at = case
    sc = scene(W, H, seed)
    K = sc.intrinsics()
    D, C, P = frames(sc, n, noise, drop, zero_at)
    vp = volume_params(W, H, filt)
    tp = recons.default_params(width=tw, height=th)
    vol = tsdf.TsdfVolume(vp)
    tr = recons.Tracker(vol, tp)
    got = tr.frames(D, C, K, P[0])
    ora = rb.OracleTracker(vp, tp)
    lost = 0
    for i in range(n):
        m = tsdf.bilateral_filter(D[i], 1000.0, 2.0, 0.05) if filt else rb.metres(D[i])
        o = ora.frame(m, C[i], K, P[0])
        g = got[i]
        assert g["cam2world"].tobytes() == o["cam2world"].tobytes(), (i, g, o)
        for k in ("iterations", "pairs", "valid_pixels", "lost"):
            assert g[k] == o[k], (i, k, g[k], o[k])
        assert np.float64(g["residual_ss"]).tobytes() == np.float64(o["residual_ss"]).tobytes(), i
        assert np.float64(g["rms"]).tobytes() == np.float64(o["rms"]).tobytes(), i
        lost += g["lost"]
    assert lost == (zero_at is not None)
    if zero_at is not None:
        assert got[zero_at]["lost"] == 1
    gx, gv = vol.download_blocks()
    ox, ov = ora.export()
    assert gx.tobytes() == ox.tobytes() and gv.tobytes() == ov.tobytes()
    mx, mc, mt = vol.extract_mesh()
    ox_, oc_, ot_ = ora.extract_mesh()
    assert mx.tobytes() == ox_.tobytes() and mc.tobytes() == oc_.tobytes() and mt.astype(np.uint32).tobytes() == ot_.tobytes()
    te, re = rb.pose_errors([g["cam2world"] for g in got], P)
    assert te <= 0.01 and re <= 0.5, (te, re)
    st = tr.stats()
    assert st["frames"] == n and st["kernel_launches"] > 0


def test_resolution_not_a_power_of_two_divisor_is_refused(built):
    vol = tsdf.TsdfVolume(volume_params(320, 240, 0))
    for w, h in ((200, 150), (160, 240), (640, 480)):
        with pytest.raises(ScnError) as e:
            recons.Tracker(vol, recons.default_params(width=w, height=h))
        assert e.value.code == -1


def test_full_heap_is_a_capacity_error(built):
    sc = scene(160, 120, 2)
    D, C, P = frames(sc, 3, 0.0, 0.0)
    vol = tsdf.TsdfVolume(volume_params(160, 120, 0, max_blocks=64))
    tr = recons.Tracker(vol, recons.default_params(width=160, height=120))
    with pytest.raises(ScnError) as e:
        tr.frames(D, C, sc.intrinsics(), P[0])
    assert e.value.code == -5


def test_missing_parameter_file_is_an_io_error(built, tmp_path):
    with pytest.raises(ScnError) as e:
        recons.params_from_file(os.path.join(str(tmp_path), "missing.txt"))
    assert e.value.code == -3


# ---------------------------------------------------------------------------------------------- the `recons` stage: .sens -> .ply + poses
import ctypes as C  # noqa: E402
import shutil  # noqa: E402
import struct  # noqa: E402
import subprocess  # noqa: E402

from scannet_b200._lib import check, lib  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
PARAMS = [os.path.join(GOLD, "zParametersScanNet.txt"), os.path.join(GOLD, "zParametersBundlingScanNet.txt")]
BIN = os.path.join(ROOT, "scannet_b200", "bin")


def pose_offsets(path):
    """Byte offsets of every frame's 64-byte pose in a .sens v4 file."""
    b = open(path, "rb").read()
    o = 4
    (nl,) = struct.unpack_from("<Q", b, o); o += 8 + nl + 4 * 64 + 8 + 16 + 4
    (n,) = struct.unpack_from("<Q", b, o); o += 8
    offs = []
    for _ in range(n):
        offs.append(o)
        cb, db = struct.unpack_from("<QQ", b, o + 64 + 16)
        o += 64 + 32 + cb + db
    return b, offs


def masked(path):
    b, offs = pose_offsets(path)
    b = bytearray(b)
    poses = []
    for o in offs:
        poses.append(np.frombuffer(bytes(b[o:o + 64]), "<f4").reshape(4, 4).copy())
        b[o:o + 64] = b"\0" * 64
    return bytes(b), np.array(poses)


def cli_params():
    p = tsdf.default_params(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02)
    tp = recons.default_params()
    for f in PARAMS:
        tsdf.params_from_file(f, p); recons.params_from_file(f, tp)
    return p, tp


@pytest.fixture(scope="module")
def capture(tmp_path_factory):
    """48 frames at 640x480 (tracking 320x240), 1 mm noise, 2 % dropouts; as a converter writes it (identity after frame 0) and with
    the generator's poses."""
    d = tmp_path_factory.mktemp("recons")
    sc = scene(640, 480, 2)
    D, C_, P = frames(sc, 48, 1.0, 0.02)
    conv = P.copy(); conv[1:] = np.eye(4, dtype=np.float32)
    synth.write_sens(str(d / "scene.sens"), D, C_, conv, sc.intrinsics(), depth_comp=1, color_comp=0)
    synth.write_sens(str(d / "gt.sens"), D, C_, P, sc.intrinsics(), depth_comp=1, color_comp=0)
    return d, sc, D, C_, P


def test_recons_cli_writes_poses_and_mesh(built, capture):
    d, sc, D, C_, P = capture
    src = str(d / "scene.sens"); work = str(d / "work.sens")
    shutil.copyfile(src, work)
    r = subprocess.run([os.path.join(BIN, "recons")] + PARAMS + [work], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "tracked 48 of 48 frames" in r.stdout
    # only the pose fields changed
    before, _ = masked(src); after, poses = masked(work)
    assert before == after
    te, re = rb.pose_errors(poses, P)
    assert te <= 0.01 and re <= 0.5, (te, re)
    # <base>.ply byte-identical to the handle path
    p, tp = cli_params()
    p.width, p.height, p.batch_frames = 640, 480, 1
    vol = tsdf.TsdfVolume(p)
    got = recons.Tracker(vol, tp).frames(D, C_, sc.intrinsics(), P[0])
    assert np.array([g["cam2world"] for g in got]).tobytes() == poses.tobytes()
    xyz, rgb, tri = vol.extract_mesh()
    xyz, rgb, tri = (np.ascontiguousarray(a) for a in (xyz, rgb, tri.astype(np.uint32)))
    ref = str(d / "handle.ply")
    check(lib().scn_mesh_save_ply(ref.encode(), xyz.ctypes.data_as(C.c_void_p), rgb.ctypes.data_as(C.c_void_p), C.c_uint64(len(xyz)),
                                  tri.ctypes.data_as(C.c_void_p), C.c_uint64(len(tri))))
    assert open(str(d / "work.ply"), "rb").read() == open(ref, "rb").read()
    # fuse on the rewritten file against fuse on the generator's poses
    from scipy.spatial import cKDTree
    for s in ("work", "gt"):
        r = subprocess.run([os.path.join(BIN, "fuse"), PARAMS[0], str(d / f"{s}.sens") if s == "work" else str(d / "gt.sens"),
                            str(d / f"{s}_vh.ply")], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
    a = synth.read_ply(str(d / "work_vh.ply"))[0]; g = synth.read_ply(str(d / "gt_vh.ply"))[0]
    dist = cKDTree(g).query(a)[0]
    # the bulk of the surface agrees to well under 2 cm; a few fringe vertices (where one mesh has a sliver the other lacks) do not
    assert len(a) > 10000 and np.percentile(dist, 99.9) <= 0.02 and (dist > 0.02).mean() < 1e-3, (len(a), np.percentile(dist, 99.9), dist.max())
    print(f"fused on tracked poses vs on generator poses: {len(a)} vertices, 99.9 % within {np.percentile(dist, 99.9) * 100:.2f} cm, "
          f"{int((dist > 0.02).sum())} beyond 2 cm, max {dist.max() * 100:.2f} cm")


def test_recons_scene_report_and_phases(built, capture):
    d, sc, D, C_, P = capture
    p, tp = cli_params()
    rep = recons.recons_scene(str(d / "scene.sens"), str(d / "r.ply"), str(d / "r.sens"), p, tp)
    assert rep["status"] == 0 and rep["frames"] == 48 and rep["frames_lost"] == 0 and rep["mesh_faces"] > 0
    assert rep["icp_ms"] > 0 and rep["raycast_ms"] > 0 and rep["integrate_ms"] > 0 and rep["filter_pyramid_ms"] > 0
    assert rep["kernel_launches"] > 48 * 19
    assert masked(str(d / "r.sens"))[0] == masked(str(d / "scene.sens"))[0]


def test_recons_full_heap_leaves_the_sens_unchanged(built, capture, tmp_path):
    d = capture[0]
    work = str(tmp_path / "small.sens"); shutil.copyfile(str(d / "scene.sens"), work)
    before = open(work, "rb").read()
    p, tp = cli_params()
    p.max_blocks = 64
    with pytest.raises(ScnError) as e:
        recons.recons_scene(work, str(tmp_path / "small.ply"), None, p, tp)
    assert e.value.code == -5
    assert open(work, "rb").read() == before and not os.path.exists(str(tmp_path / "small.ply"))


def test_recons_missing_sens_is_an_io_error(built, tmp_path):
    with pytest.raises(ScnError) as e:
        recons.recons_scene(str(tmp_path / "missing.sens"), None)
    assert e.value.code == -3
