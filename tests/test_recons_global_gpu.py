"""`recons --global` (scn_recons_scene_global, DESIGN.md §6k) on a .sens: only the pose fields change and lost frames stay -inf;
the keyframe poses equal the handle path (Tracker, then GlobalOptimizer on the same frames) bit for bit and the other frames follow
their keyframe by the stated propagation; the PLY is byte-identical to scn_fuse_scene on the written .sens; the ATE stays within the
tracker's bounds; and a refused call writes nothing."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import recons_bindings as rb
from scannet_b200 import ScnError, recons, synth, tsdf
from scannet_b200._lib import check, lib
from test_recons_gpu import BIN, PARAMS, cli_params, frames, masked, scene

pytestmark = pytest.mark.gpu


def global_params(**over):
    gp = recons.global_default_params()
    for f in PARAMS:
        recons.global_params_from_file(f, gp)
    for k, v in over.items():
        setattr(gp, k, v)
    return gp


def write_capture(d, W, H, n, zero_at, seed=2):
    sc = scene(W, H, seed)
    D, C_, P = frames(sc, n, 1.0, 0.02, zero_at)
    conv = P.copy(); conv[1:] = np.eye(4, dtype=np.float32)         # as a converter writes it: identity after frame 0
    path = os.path.join(d, "scene.sens")
    synth.write_sens(path, D, C_, conv, sc.intrinsics(), depth_comp=1, color_comp=0)
    return path, sc, D, C_, P


def handle_path(sc, D, C_, P, gp):
    """Tracker then GlobalOptimizer on the same frames; the expected poses of every frame"""
    p, tp = cli_params()
    p.width, p.height, p.batch_frames = sc.W, sc.H, 1
    vol = tsdf.TsdfVolume(p)
    got = recons.Tracker(vol, tp).frames(D, C_, sc.intrinsics(), P[0])
    T = np.array([g["cam2world"] for g in got])
    lost = [g["lost"] for g in got]
    kf = recons.keyframe_indices(lost, gp.submap_size)
    opt = recons.GlobalOptimizer(vol, gp)
    opt.add_keyframes(D[kf], T[kf], sc.intrinsics())
    K, rep = opt.solve()
    of_submap = {f // gp.submap_size: k for k, f in enumerate(kf)}
    out = T.copy()
    if not rep["rejected"]:
        for f in range(len(D)):
            if lost[f]:
                continue
            k = of_submap[f // gp.submap_size]
            out[f] = K[k] if kf[k] == f else recons.propagate(T[kf[k]], K[k], T[f])
    return T, out, rep


def fuse_ply(path, out):
    p, _ = cli_params()
    check(lib().scn_fuse_scene(path.encode(), out.encode(), C.byref(p), 0, None, None))
    return open(out, "rb").read()


def test_recons_global_cli_on_a_capture(built, tmp_path):
    d = str(tmp_path)
    src, sc, D, C_, P = write_capture(d, 640, 480, 48, zero_at=20)
    work = os.path.join(d, "work.sens"); shutil.copyfile(src, work)
    r = subprocess.run([os.path.join(BIN, "recons"), "--global"] + PARAMS + [work], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "global optimisation: 5 keyframes" in r.stdout, r.stdout
    before, _ = masked(src); after, poses = masked(work)
    assert before == after                                          # only the pose fields changed
    assert np.isneginf(poses[20]).all()                             # the lost frame keeps -inf
    T, want, rep = handle_path(sc, D, C_, P, global_params())
    assert poses.tobytes() == want.tobytes()
    assert open(os.path.join(d, "work.ply"), "rb").read() == fuse_ply(work, os.path.join(d, "fused.ply"))
    keep = [f for f in range(48) if f != 20]
    te, re = rb.pose_errors(poses[keep], P[keep]); te0, re0 = rb.pose_errors(T[keep], P[keep])
    print(f"48 frames: ATE {te0 * 1000:.2f} mm / {re0:.3f} deg tracked, {te * 1000:.2f} mm / {re:.3f} deg after --global "
          f"({rep['edges_consecutive']}+{rep['edges_loop']} edges, rejected {rep['rejected']})")
    assert te <= 0.01 and re <= 0.5


def test_recons_global_on_a_300_frame_orbit(built, tmp_path):
    d = str(tmp_path)
    src, sc, D, C_, P = write_capture(d, 320, 240, 300, zero_at=None)
    plain = os.path.join(d, "plain.sens"); shutil.copyfile(src, plain)
    p, tp = cli_params()
    recons.recons_scene(plain, os.path.join(d, "plain.ply"), None, p, tp)
    rep, grep = recons.recons_scene_global(src, os.path.join(d, "g.ply"), os.path.join(d, "g.sens"), p, tp, global_params())
    assert grep["keyframes"] == 30 and grep["edges_loop"] > 0
    g = masked(os.path.join(d, "g.sens")); pl = masked(plain)
    assert g[0] == masked(src)[0]
    T, want, _ = handle_path(sc, D, C_, P, global_params())
    assert g[1].tobytes() == want.tobytes()
    assert open(os.path.join(d, "g.ply"), "rb").read() == fuse_ply(os.path.join(d, "g.sens"), os.path.join(d, "fused.ply"))
    te, re = rb.pose_errors(g[1], P); te0, re0 = rb.pose_errors(pl[1], P)
    print(f"300 frames: ATE {te0 * 1000:.2f} mm / {re0:.3f} deg tracked, {te * 1000:.2f} mm / {re:.3f} deg after --global; "
          f"{grep['edges_consecutive']}+{grep['edges_loop']} edges, {grep['edges_removed']} removed, rejected {grep['rejected']}, "
          f"RMS {grep['rms_before'] * 1000:.2f} -> {grep['rms_after'] * 1000:.2f} mm")
    assert te <= 0.01 and re <= 0.5


def test_recons_global_capacity_writes_nothing(built, tmp_path):
    d = str(tmp_path)
    src, sc, D, C_, P = write_capture(d, 320, 240, 48, zero_at=None)
    before = open(src, "rb").read()
    p, tp = cli_params()
    with pytest.raises(ScnError) as e:
        recons.recons_scene_global(src, os.path.join(d, "x.ply"), None, p, tp, global_params(max_keyframes=2))
    assert e.value.code == -5
    assert open(src, "rb").read() == before and not os.path.exists(os.path.join(d, "x.ply"))


def test_recons_global_bad_keyframe_resolution_is_refused(built, tmp_path):
    d = str(tmp_path)
    src, sc, D, C_, P = write_capture(d, 320, 240, 12, zero_at=None)
    p, tp = cli_params()
    with pytest.raises(ScnError) as e:
        recons.recons_scene_global(src, os.path.join(d, "x.ply"), None, p, tp, global_params(width=60, height=45))
    assert e.value.code == -1 and not os.path.exists(os.path.join(d, "x.ply"))
