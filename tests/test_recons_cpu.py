"""Tracking spec v1 (DESIGN.md §6j) on the CPU oracle: the linear system against a float64 numpy statement, the fixed reduction
tree, the Cayley update, pose recovery, the accuracy bound on a 300-frame loop, and the loss rules."""
import types

import numpy as np
from scipy.linalg import expm

import recons_bindings as rb
from scannet_b200 import synth


def vparams(W, H, **over):
    p = dict(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02, depth_min=0.1, depth_max=6.0, max_integration_distance=4.0,
             weight_sample=1, weight_max=255, width=W, height=H, depth_shift=1000.0)
    p.update(over)
    return types.SimpleNamespace(**p)


def tparams(W=320, H=240):
    return types.SimpleNamespace(width=W, height=H, dist_thresh=0.15, normal_thresh=0.95, ray_increment_factor=0.8)


def scene(W=320, H=240, size=(5.0, 4.0, 3.0), n_spheres=10, seed=2):
    return synth.BoxRoomScene(size=size, n_spheres=n_spheres, seed=seed, width=W, height=H, fx=synth.FX * W / 640, fy=synth.FY * H / 480,
                              cx=(W - 1) / 2, cy=(H - 1) / 2)


def perturb(T, rot_deg, trans):
    w = np.radians(rot_deg) * np.array([0.3, -0.8, 0.52]) / np.linalg.norm([0.3, -0.8, 0.52])
    S = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    E = np.eye(4); E[:3, :3] = expm(S); E[:3, 3] = trans
    return (T.astype(np.float64) @ E).astype(np.float32)


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def test_system_matches_float64_statement_and_fixed_tree():
    sc = scene()
    K = sc.intrinsics()
    P0 = sc.orbit_pose(0, 300, height=2.2)
    d0, c0 = sc.render(P0)
    d1, _ = sc.render(perturb(P0, 0.5, [0.01, -0.005, 0.008]))
    tr = rb.OracleTracker(vparams(320, 240), tparams())
    tr.frame(rb.metres(d0), c0, K, P0)
    tr.set_frame(rb.metres(d1), K)
    D = np.eye(4, dtype=np.float32)
    D[:3, 3] = [0.002, -0.001, 0.003]
    f = np.float32
    for k in range(3):
        s, n = tr.system(k, D)
        terms, paired = tr.terms(k, D)
        assert n == int(paired.sum()) > 300
        # float32 association restated in numpy, then the system in float64
        v, nrm, mv, mn = tr.maps(k)
        w, h = tr.level_size(k)
        sc_ = f(1.0) / f(1 << k)
        fx, fy = f(K[0, 0]) * sc_, f(K[1, 1]) * sc_
        cx, cy = (f(K[0, 2]) + f(0.5)) * sc_ - f(0.5), (f(K[1, 2]) + f(0.5)) * sc_ - f(0.5)
        Df = D[:3, :4].astype(np.float32)
        p = v.reshape(-1, 4); pn = nrm.reshape(-1, 4)
        T = [((Df[i, 0] * p[:, 0] + Df[i, 1] * p[:, 1]) + Df[i, 2] * p[:, 2]) + Df[i, 3] for i in range(3)]
        Rn = [(Df[i, 0] * pn[:, 0] + Df[i, 1] * pn[:, 1]) + Df[i, 2] * pn[:, 2] for i in range(3)]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = np.rint((T[0] / T[2]) * fx + cx); vv = np.rint((T[1] / T[2]) * fy + cy)
        ok = (pn[:, 3] > 0) & (T[2] > 0) & (u >= 0) & (u <= w - 1) & (vv >= 0) & (vv <= h - 1)
        j = np.where(ok, np.nan_to_num(vv) * w + np.nan_to_num(u), 0).astype(np.int64)
        q = mv.reshape(-1, 4)[j]; nq = mn.reshape(-1, 4)[j]
        d = [T[i] - q[:, i] for i in range(3)]
        ok &= nq[:, 3] > 0
        ok &= (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] <= f(0.15) * f(0.15)
        ok &= (Rn[0] * nq[:, 0] + Rn[1] * nq[:, 1]) + Rn[2] * nq[:, 2] >= f(0.95)
        assert (ok == (paired == 1)).all()
        Tp = np.stack(T, 1)[ok].astype(np.float64); Q = q[ok, :3].astype(np.float64); N = nq[ok, :3].astype(np.float64)
        r = ((Tp - Q) * N).sum(1)
        J = np.concatenate([np.cross(Tp, N), N], 1)
        A = J.T @ J; b = J.T @ r
        ref = np.concatenate([A[np.triu_indices(6)], b, [r @ r]])
        assert np.allclose(s, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max()), np.abs(s - ref).max()
        # the tree: warps of 32 by a halving tree, 8 warp sums by a halving tree, slots added in order
        npx = w * h
        ncta = (npx + 255) // 256
        t = np.zeros((ncta * 256, 28)); t[:npx] = terms
        t = t.reshape(ncta, 8, 32, 28)
        for st in (16, 8, 4, 2, 1):
            t[:, :, :st] = t[:, :, :st] + t[:, :, st:2 * st]
        wsum = t[:, :, 0].copy()
        for st in (4, 2, 1):
            wsum[:, :st] = wsum[:, :st] + wsum[:, st:2 * st]
        tot = np.zeros(28)
        for c in range(ncta):
            tot = tot + wsum[c, 0]
        assert tot.tobytes() == s.tobytes()


def test_cayley_orthonormal_and_second_order():
    rng = np.random.default_rng(1)
    for scale in (1e-1, 1e-2, 1e-3):
        for _ in range(20):
            w = rng.normal(size=3) * scale
            R = rb.cayley(w)
            assert np.abs(R.T @ R - np.eye(3)).max() < 1e-12
            assert abs(np.linalg.det(R) - 1) < 1e-12
            err = np.abs(R - expm(skew(w))).max()
            assert err <= 0.2 * np.linalg.norm(w) ** 3 + 1e-15


def test_solve_refuses_an_indefinite_system():
    s = np.zeros(28)
    assert rb.solve(s, 0) is None
    A = np.diag([1.0, 2, 3, 4, 5, 6]); b = np.arange(6.0)
    iu = np.triu_indices(6)
    x = rb.solve(np.concatenate([A[iu], b, [0.0]]), 0)
    assert np.allclose(x, -b / np.diag(A), rtol=1e-15)


def test_recovers_a_perturbed_pose_noise_free():
    """Depth is stored in whole millimetres and the model comes from a 1 cm volume, so the frame and the model disagree by a few
    tenths of a millimetre: the pose is recovered to 2e-4 m / 5e-4 rad (measured 1.1e-4 m / 2.5e-4 rad), not 1e-4 (DESIGN.md §6j)."""
    sc = scene()
    K = sc.intrinsics()
    P0 = sc.orbit_pose(0, 300, height=2.2)
    d0, c0 = sc.render(P0)
    tr = rb.OracleTracker(vparams(320, 240), tparams())
    tr.frame(rb.metres(d0), c0, K, P0)
    P1 = perturb(P0, 1.0, [0.02, -0.01, 0.015])
    d1, c1 = sc.render(P1)
    r = tr.frame(rb.metres(d1), c1, K)
    assert not r["lost"]
    te, re = rb.pose_errors([r["cam2world"]], [P1])
    assert te <= 2e-4 and np.radians(re) <= 5e-4, (te, re)


def run_loop(sc, n, K, noise=1.0, drop=0.02):
    tr = rb.OracleTracker(vparams(sc.W, sc.H), tparams(sc.W, sc.H))
    est, gt, res = [], [], []
    for i in range(n):
        P = sc.orbit_pose(i, 300, height=2.2)
        d, c = sc.render(P, noise_mm=noise, drop=drop, frame_seed=i)
        r = tr.frame(rb.metres(d), c, K, P)
        est.append(r["cam2world"]); gt.append(P); res.append(r)
    return tr, est, gt, res


def test_accuracy_on_a_300_frame_loop():
    """1 mm noise, 2 % dropouts, 1 cm voxels, 320x240: translation RMS <= 1 cm, rotation <= 0.5 deg against the generator."""
    sc = scene()
    _, est, gt, res = run_loop(sc, 300, sc.intrinsics())
    assert not any(r["lost"] for r in res)
    te, re = rb.pose_errors(est, gt)
    assert te <= 0.01 and re <= 0.5, (te, re)


def test_lost_frames_are_not_integrated_and_tracking_resumes():
    sc = scene(160, 120)
    K = sc.intrinsics()
    other = synth.BoxRoomScene(size=(5.0, 4.0, 3.0), n_spheres=10, seed=2, width=160, height=120, fx=sc.fx, fy=sc.fy, cx=sc.cx, cy=sc.cy)
    far = np.eye(4, dtype=np.float32)
    far[:3, :3] = np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], np.float32)      # looking straight up from a corner of the floor
    far[:3, 3] = [0.4, 0.4, 0.3]
    d_far, c_far = other.render(far)
    snapshots = {}

    def hook(i, d, c):
        if i == 12:
            return np.zeros_like(d), c
        if i == 20:
            return d_far, c_far
        return d, c

    tr = rb.OracleTracker(vparams(160, 120), tparams(160, 120))
    est, gt, res = [], [], []
    for i in range(40):
        P = sc.orbit_pose(i, 300, height=2.2)
        d, c = sc.render(P, noise_mm=1.0, drop=0.02, frame_seed=i)
        d, c = hook(i, d, c)
        if i in (12, 20):
            snapshots[i] = tr.export()
        r = tr.frame(rb.metres(d), c, K, P)
        if i in (12, 20):
            after = tr.export()
            assert r["lost"] == 1 and np.isneginf(r["cam2world"]).all(), (i, r)
            assert after[0].tobytes() == snapshots[i][0].tobytes() and after[1].tobytes() == snapshots[i][1].tobytes()
        else:
            assert r["lost"] == 0, (i, r)
            est.append(r["cam2world"]); gt.append(P)
    te, re = rb.pose_errors(est, gt)
    assert te <= 0.01 and re <= 0.5, (te, re)


def test_report_bindings_match_the_library_structs():
    import ctypes as C
    from scannet_b200 import recons
    from scannet_b200._lib import lib
    lib().scn_track_frame_sizeof.restype = C.c_size_t
    lib().scn_recons_report_sizeof.restype = C.c_size_t
    assert lib().scn_track_frame_sizeof() == C.sizeof(recons.TrackFrame) == C.sizeof(rb.TrackFrame)
    assert lib().scn_recons_report_sizeof() == C.sizeof(recons.ReconsReport)


def test_pyramid_and_normals_on_a_designed_depth_map():
    """Independent of the oracle's own maps: a tilted plane z = a + b x + c y at 16x12 (tracking = depth resolution) with two holes.
    Reductions average the valid pixels of each 2x2; normals are the normalised dv x du of the plane; holes make their neighbours
    invalid at level 0."""
    W, H = 16, 12
    K = np.eye(4, dtype=np.float32); K[0, 0] = K[1, 1] = 20.0; K[0, 2] = 7.5; K[1, 2] = 5.5
    # a plane in camera space n.X = d seen by the pinhole: depth(x, y) = d / (n . ((x-cx)/f, (y-cy)/f, 1))
    n = np.array([0.2, -0.1, -1.0]); n /= np.linalg.norm(n); d = -2.0
    ys, xs = np.mgrid[0:H, 0:W]
    ray = np.stack([(xs - 7.5) / 20.0, (ys - 5.5) / 20.0, np.ones_like(xs, float)], -1)
    depth = (d / (ray @ n)).astype(np.float32)
    depth[3, 4] = -np.inf; depth[8, 9] = -np.inf
    tr = rb.OracleTracker(vparams(W, H), tparams(W, H))
    assert tr.set_frame(depth, K) == (W - 2) * (H - 2) - 2 * 5 + 0
    v0, n0, _, _ = tr.maps(0)
    ok = n0[..., 3] > 0
    assert not ok[3, 4] and not ok[2, 4] and not ok[3, 5] and not ok[8, 8] and not ok[9, 9]
    assert np.abs(n0[ok][:, :3] - n).max() < 2e-4                 # dv x du points towards the camera: n_z < 0
    assert np.abs(v0[ok][:, 2] - depth[ok]).max() == 0
    v1, _, _, _ = tr.maps(1)
    blk = depth.reshape(H // 2, 2, W // 2, 2).transpose(0, 2, 1, 3).reshape(H // 2, W // 2, 4).astype(np.float64)
    fin = np.isfinite(blk)
    ref = np.where(fin, blk, 0).sum(-1) / fin.sum(-1)
    assert np.abs(v1[..., 2] - ref).max() < 1e-6


def test_raycast_depth_of_a_wall_matches_its_distance():
    """The model depth of a fronto-parallel wall, integrated from one frame, against the analytic distance."""
    W, H = 64, 48
    K = np.eye(4, dtype=np.float32); K[0, 0] = K[1, 1] = 60.0; K[0, 2] = 31.5; K[1, 2] = 23.5
    depth = np.full((H, W), 1234, np.uint16)
    tr = rb.OracleTracker(vparams(W, H), tparams(W, H))
    r = tr.frame(rb.metres(depth), None, K, np.eye(4, dtype=np.float32))
    assert not r["lost"]
    md = tr.model_depth()
    ok = np.isfinite(md)
    assert ok[4:-4, 4:-4].all()
    assert np.abs(md[ok] - 1.234).max() < 1e-3


def test_an_empty_first_frame_does_not_seed_the_model():
    sc = scene(160, 120)
    K = sc.intrinsics()
    tr = rb.OracleTracker(vparams(160, 120), tparams(160, 120))
    P = [sc.orbit_pose(i, 300, height=2.2) for i in range(4)]
    r0 = tr.frame(rb.metres(np.zeros((120, 160), np.uint16)), None, K, P[1])
    assert r0["lost"] == 1 and np.isneginf(r0["cam2world"]).all() and tr.export()[0].shape[0] == 0
    r1 = tr.frame(rb.metres(sc.render(P[1])[0]), None, K, P[1])            # the seed takes the stored first pose
    assert r1["lost"] == 0 and r1["cam2world"].tobytes() == P[1].tobytes()
    for i in (2, 3):
        r = tr.frame(rb.metres(sc.render(P[i])[0]), None, K, P[1])
        assert r["lost"] == 0
        te, re = rb.pose_errors([r["cam2world"]], [P[i]])
        assert te < 2e-3 and re < 0.1
