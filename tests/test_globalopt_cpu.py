"""The global optimisation oracle (oracle/globalopt_oracle.c, DESIGN.md §6k) against float64 statements of its per-edge sums, its
assembled system and its PCG solution; drift recovery on a closed loop; verification of a keyframe from another scene; the
parameter file and the report struct.  No GPU."""
import ctypes as C
import os

import numpy as np
import pytest

import globalopt_bindings as gb
import recons_bindings as rb
from scannet_b200 import recons

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- a float64 statement of one edge's sums ------------------------------------------------------------------------------------
# The keyframe maps and the association are restated in binary32 numpy in the spec's order, so that the pairs are the oracle's;
# the products and the sums are then formed in float64 in numpy's own order.
def reduce2(d):
    q = np.stack([d[0::2, 0::2], d[0::2, 1::2], d[1::2, 0::2], d[1::2, 1::2]])
    ok = q != -np.inf
    z = np.where(ok, q, np.float32(0))
    n = ok.sum(0).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        m = ((z[0] + z[1]) + (z[2] + z[3])) / n
    return np.where(n > 0, m, np.float32(-np.inf)).astype(np.float32)


def keyframe_maps(metres, K, p, s):
    d = np.where((metres >= np.float32(p.depth_min)) & (metres <= np.float32(p.depth_max)), metres, np.float32(-np.inf)).astype(np.float32)
    for _ in range(s):
        d = reduce2(d)
    sc = np.float32(1.0) / np.float32(1 << s)
    fx, fy = np.float32(K[0, 0]) * sc, np.float32(K[1, 1]) * sc
    cx = (np.float32(K[0, 2]) + np.float32(0.5)) * sc - np.float32(0.5)
    cy = (np.float32(K[1, 2]) + np.float32(0.5)) * sc - np.float32(0.5)
    ifx, ify = np.float32(1) / fx, np.float32(1) / fy
    H, W = d.shape
    xs, ys = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32))
    ok = d != -np.inf
    dz = np.where(ok, d, np.float32(0))
    V = np.stack([((xs - cx) * ifx) * dz, ((ys - cy) * ify) * dz, dz], -1).astype(np.float32)
    N = np.zeros_like(V)
    nok = np.zeros((H, W), bool)
    c = ok[1:-1, 1:-1] & ok[1:-1, 2:] & ok[1:-1, :-2] & ok[2:, 1:-1] & ok[:-2, 1:-1]
    u = V[1:-1, 2:] - V[1:-1, :-2]
    v = V[2:, 1:-1] - V[:-2, 1:-1]
    cr = np.stack([v[..., 1] * u[..., 2] - v[..., 2] * u[..., 1], v[..., 2] * u[..., 0] - v[..., 0] * u[..., 2],
                   v[..., 0] * u[..., 1] - v[..., 1] * u[..., 0]], -1)
    ln = np.sqrt((cr[..., 0] * cr[..., 0] + cr[..., 1] * cr[..., 1]) + cr[..., 2] * cr[..., 2])
    good = c & (ln > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        N[1:-1, 1:-1] = np.where(good[..., None], cr / ln[..., None], 0).astype(np.float32)
    nok[1:-1, 1:-1] = good
    return V.reshape(-1, 3), N.reshape(-1, 3), nok.reshape(-1), (W, H, fx, fy, cx, cy)


def dot3(M, r, p):
    return (M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1]) + M[r, 2] * p[:, 2]


def edge_sums_f64(mi, mj, Ti, Tj, p):
    Vi, Ni, oki, (W, H, fx, fy, cx, cy) = mi
    Vj, Nj, okj, _ = mj
    Di, Dj = Ti.astype(np.float64), Tj.astype(np.float64)
    M = (Di[:3, :3].T @ Dj[:3, :]).astype(np.float64)
    M[:, 3] -= Di[:3, :3].T @ Di[:3, 3]
    M = M.astype(np.float32)    # the oracle rounds the binary64 product once; identical here unless a rounding tie differs
    t = np.stack([dot3(M, r, Vj) + M[r, 3] for r in range(3)], -1).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        u = np.rint((t[:, 0] / t[:, 2]) * fx + cx)
        v = np.rint((t[:, 1] / t[:, 2]) * fy + cy)
    ok = okj & (t[:, 2] > 0) & (u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1)
    idx = np.where(ok, np.nan_to_num(v) * W + np.nan_to_num(u), 0).astype(np.int64)
    ok &= oki[idx]
    q, nq = Vi[idx], Ni[idx]
    d = (t - q).astype(np.float32)
    ok &= ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) <= np.float32(p.dist_thresh) * np.float32(p.dist_thresh)
    rn = np.stack([dot3(M, r, Nj) for r in range(3)], -1).astype(np.float32)
    ok &= ((rn[:, 0] * nq[:, 0] + rn[:, 1] * nq[:, 1]) + rn[:, 2] * nq[:, 2]) >= np.float32(p.normal_thresh)
    r = ((d[:, 0] * nq[:, 0] + d[:, 1] * nq[:, 1]) + d[:, 2] * nq[:, 2])[ok].astype(np.float64)
    w = Vj[ok].astype(np.float64) @ Dj[:3, :3].T + Dj[:3, 3]
    nw = nq[ok].astype(np.float64) @ Di[:3, :3].T
    a = np.concatenate([np.cross(w, nw), nw], 1)
    S = a.T @ a
    iu = np.triu_indices(6)
    return np.concatenate([S[iu], a.T @ r, [r @ r]]), int(ok.sum())


def designed(n, W=160, H=120, gp=None):
    sc = gb.scene(W, H)
    D, P, Q = gb.loop_keyframes(sc, n, noise_mm=0.5)
    p = gp or recons.global_default_params(width=W // 2, height=H // 2)
    o = gb.OracleGlobal(p, W, H)
    M = [rb.metres(D[k]) for k in range(n)]
    for k in range(n):
        o.add_keyframe(M[k], sc.intrinsics(), Q[k])
    return sc, o, p, M, P, Q


@pytest.mark.parametrize("n", [2, 6])
def test_edge_sums_match_float64(built, n):
    sc, o, p, M, P, Q = designed(n)
    maps = [keyframe_maps(M[k], sc.intrinsics(), p, 1) for k in range(n)]
    checked = 0
    for i in range(n):
        for j in range(i + 1, n):
            s, pairs = o.edge_system(i, j)
            ref, rpairs = edge_sums_f64(maps[i], maps[j], Q[i], Q[j], p)
            assert pairs == rpairs, (i, j)
            if pairs:
                np.testing.assert_allclose(s, ref, rtol=1e-5, atol=1e-7 * np.abs(ref).max())   # a is formed in binary32
                checked += 1
    assert checked >= n - 1


@pytest.mark.parametrize("n", [2, 6])
def test_assembled_system_and_pcg_match_float64(built, n):
    sc, o, p, M, P, Q = designed(n)
    edges = [(i, j) for i in range(n) for j in range(i + 1, n)]
    H, rhs, free, x = o.first_system(edges, 6 * n + 6)
    # H and -g from the per-edge sums, in float64
    Hr = np.zeros_like(H); g = np.zeros(6 * n)
    pk = np.zeros(n)
    iu = np.triu_indices(6)
    for (i, j) in edges:
        s, pairs = o.edge_system(i, j)
        S = np.zeros((6, 6)); S[iu] = s[:21]; S = S + np.triu(S, 1).T
        for a, b, sg in ((i, i, 1), (j, j, 1), (i, j, -1), (j, i, -1)):
            Hr[6 * a:6 * a + 6, 6 * b:6 * b + 6] += sg * S
        g[6 * j:6 * j + 6] += s[21:27]; g[6 * i:6 * i + 6] -= s[21:27]
        pk[i] += pairs; pk[j] += pairs
    Hr += np.diag(np.repeat(pk * 2.0 ** -13, 6))
    np.testing.assert_allclose(H, Hr, rtol=1e-12, atol=1e-12 * np.abs(Hr).max())
    assert not free[0] and free[1:].all()
    fm = np.repeat(free, 6)
    np.testing.assert_allclose(rhs[fm], -g[fm], rtol=1e-12, atol=1e-12 * np.abs(g).max())
    assert (rhs[~fm] == 0).all()
    ref = np.linalg.solve(Hr[np.ix_(fm, fm)], -g[fm])
    np.testing.assert_allclose(x[fm], ref, rtol=1e-6, atol=1e-9 * np.abs(ref).max())
    assert (x[~fm] == 0).all()


def test_drift_is_recovered_on_a_closed_loop(built):
    W, H, n = 320, 240, 12
    sc = gb.scene(W, H)
    D, P, Q = gb.loop_keyframes(sc, n)
    o = gb.OracleGlobal(recons.global_default_params(), W, H)
    for k in range(n):
        assert o.add_keyframe(rb.metres(D[k]), sc.intrinsics(), Q[k]) > 1000
    poses, rep = o.solve()
    edges = {(e["i"], e["j"]): e for e in o.edges()}
    assert (0, n - 1) in edges and edges[(0, n - 1)]["loop"] and not edges[(0, n - 1)]["removed"]
    assert rep["edges_consecutive"] == n - 1 and rep["edges_loop"] >= 1 and not rep["rejected"]
    assert poses[0].tobytes() == Q[0].tobytes()
    before, after = gb.ate(Q, P), gb.ate(poses, P)
    print(f"ATE {before[0] * 1000:.1f} mm / {before[1]:.2f} deg -> {after[0] * 1000:.2f} mm / {after[1]:.3f} deg; "
          f"RMS {rep['rms_before'] * 1000:.2f} -> {rep['rms_after'] * 1000:.2f} mm, {rep['edges_loop']} loop edges")
    assert before[0] > 0.03 and after[0] <= before[0] / 5
    assert after[0] <= 0.005 and after[1] <= 0.3        # measured: 3.2 mm, 0.18 deg
    assert rep["rss_iter"][0] > rep["rss_iter"][1] > rep["rss_iter"][2] > rep["rss_after"]


def test_keyframe_from_another_scene_is_cut_loose(built):
    W, H, n, bad = 320, 240, 12, 5
    sc = gb.scene(W, H)
    D, P, Q = gb.loop_keyframes(sc, n, bad=bad)
    o = gb.OracleGlobal(recons.global_default_params(), W, H)
    for k in range(n):
        o.add_keyframe(rb.metres(D[k]), sc.intrinsics(), Q[k])
    poses, rep = o.solve()
    touching = [e for e in o.edges() if bad in (e["i"], e["j"])]
    assert touching and all(e["removed"] for e in touching)
    assert rep["edges_removed"] == len(touching) and not rep["rejected"]
    assert poses[bad].tobytes() == Q[bad].tobytes()
    keep = [k for k in range(n) if k != bad]
    assert gb.ate(poses[keep], P[keep])[0] <= 0.005


def test_too_many_removals_reject_the_result(built):
    W, H, n = 160, 120, 6
    sc, o, p, M, P, Q = designed(n, W, H, recons.global_default_params(width=80, height=60, verify_thresh=1e-4, max_removed=2))
    poses, rep = o.solve()
    assert rep["rejected"] == 1 and rep["edges_removed"] == 2 and rep["solves"] == 3
    assert poses.tobytes() == Q.tobytes()


def test_parameter_file_reads_every_global_key(built):
    p = recons.global_params_from_file(os.path.join(ROOT, "tests/golden/zParametersBundlingScanNet.txt"),
                                       recons.GlobalParams())
    assert (p.submap_size, p.max_keyframes, p.width, p.height) == (10, 2000, 80, 60)
    assert (p.dist_thresh, p.normal_thresh, p.depth_min, p.depth_max) == (np.float32(0.15), np.float32(0.95), 0.5, 4.0)
    assert (p.overlap_subsample, p.nonlin_iters, p.lin_iters, p.max_removed) == (4, 3, 150, 10)
    assert p.verify_thresh == np.float32(0.05)
    d = recons.global_default_params()
    assert bytes(d) == bytes(p)


def test_report_binding_matches_the_library_struct(built):
    from scannet_b200._lib import lib
    lib().scn_globalopt_report_sizeof.restype = C.c_size_t
    assert lib().scn_globalopt_report_sizeof() == C.sizeof(recons.GlobalReport)


def test_keyframe_selection():
    assert recons.keyframe_indices([0] * 25, 10) == [0, 10, 20]
    assert recons.keyframe_indices([1, 1, 0, 0] + [1] * 4 + [0, 1], 4) == [2, 8]
