"""ctypes bindings for the global optimisation oracle (oracle/_build/liboracle_globalopt.so, DESIGN.md §6k).  TEST INFRASTRUCTURE:
only tests/, __graft_entry__.smoke() and scripts/bench_globalopt.py import this."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle/_build/liboracle_globalopt.so")
NSUM = 28
MAX_NONLIN = 16


class OracleGlobalParams(C.Structure):
    """= scn_globalopt_params"""
    _fields_ = [("submap_size", C.c_uint32), ("max_keyframes", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32),
                ("dist_thresh", C.c_float), ("normal_thresh", C.c_float), ("depth_min", C.c_float), ("depth_max", C.c_float),
                ("overlap_subsample", C.c_uint32), ("nonlin_iters", C.c_uint32), ("lin_iters", C.c_uint32), ("verify_thresh", C.c_float),
                ("max_removed", C.c_uint32)]


class OracleGlobalReport(C.Structure):
    """the counters of scn_globalopt_report_t"""
    _fields_ = [(k, C.c_uint32) for k in ("keyframes", "edges_consecutive", "edges_loop", "edges_removed", "rejected", "solves",
                                          "nonlin_iterations", "lin_iterations")] + [
        ("pairs_before", C.c_uint64), ("pairs_after", C.c_uint64)] + [
        (k, C.c_double) for k in ("rss_before", "rss_after", "rms_before", "rms_after", "max_edge_rms")] + [
        ("rss_iter", C.c_double * MAX_NONLIN)]


COUNTERS = [k for k, _ in OracleGlobalReport._fields_ if k != "rss_iter"]

_o = None


def _lib():
    global _o
    if _o is None:
        if not os.path.exists(ORACLE):
            raise FileNotFoundError(f"{ORACLE} missing — run `make oracle` (oracle/globalopt.mk)")
        _o = C.CDLL(ORACLE)
        _o.oracle_go_create.restype = C.c_void_p
        _o.oracle_go_create.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        _o.oracle_go_destroy.argtypes = [C.c_void_p]
        _o.oracle_go_add_keyframe.argtypes = [C.c_void_p] * 4
        _o.oracle_go_solve.argtypes = [C.c_void_p] * 3
        _o.oracle_go_num_edges.argtypes = [C.c_void_p]
        _o.oracle_go_edges.argtypes = [C.c_void_p] * 7
        _o.oracle_go_edge_system.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _o.oracle_go_first_system.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
        _o.oracle_go_pcg_trace.argtypes = [C.c_void_p] * 3
    return _o


class OracleGlobal:
    """The oracle's keyframes and solve.  params: an object with the scn_globalopt_params fields; (W, H) the depth resolution."""

    def __init__(self, params, W: int, H: int):
        p = OracleGlobalParams()
        for f, _ in OracleGlobalParams._fields_:
            setattr(p, f, getattr(params, f))
        self.p = p
        self.n = 0
        self._h = _lib().oracle_go_create(C.byref(p), W, H)
        if not self._h:
            raise ValueError("keyframe resolution is not the depth resolution divided by a power of two")

    def __del__(self):
        if getattr(self, "_h", None):
            _lib().oracle_go_destroy(self._h)
            self._h = None

    def add_keyframe(self, metres_img, K, pose) -> int:
        m = np.ascontiguousarray(metres_img, np.float32)
        Kc = np.ascontiguousarray(K, np.float32)
        T = np.ascontiguousarray(pose, np.float32)
        v = _lib().oracle_go_add_keyframe(self._h, m.ctypes.data, Kc.ctypes.data, T.ctypes.data)
        if v >= 0:
            self.n += 1
        return v

    def solve(self):
        out = np.zeros((max(self.n, 1), 4, 4), np.float32)
        r = OracleGlobalReport()
        _lib().oracle_go_solve(self._h, out.ctypes.data, C.byref(r))
        d = {k: getattr(r, k) for k in COUNTERS}
        d["rss_iter"] = tuple(r.rss_iter)
        return out[:self.n], d

    def edges(self) -> list[dict]:
        ne = _lib().oracle_go_num_edges(self._h)
        a = [np.zeros(ne, np.int32) for _ in range(4)]
        pairs = np.zeros(ne, np.uint32)
        sums = np.zeros((ne, NSUM), np.float64)
        _lib().oracle_go_edges(self._h, *[x.ctypes.data for x in a], pairs.ctypes.data, sums.ctypes.data)
        return [dict(i=int(a[0][e]), j=int(a[1][e]), loop=int(a[2][e]), removed=int(not a[3][e]), pairs=int(pairs[e]),
                     rss=float(sums[e, 27]), sums=sums[e]) for e in range(ne)]

    def edge_system(self, i, j):
        """the 28 sums of (i, j) at the poses handed in and the pairs"""
        s = np.zeros(NSUM, np.float64)
        n = C.c_uint32(0)
        _lib().oracle_go_edge_system(self._h, i, j, s.ctypes.data, C.byref(n))
        return s, int(n.value)

    def first_system(self, edges, iters):
        """(dense damped H, -g, free flags, PCG solution after `iters` iterations) of the first linear system over `edges`"""
        n = self.n
        ei = np.ascontiguousarray([e[0] for e in edges], np.int32)
        ej = np.ascontiguousarray([e[1] for e in edges], np.int32)
        H = np.zeros((6 * n, 6 * n), np.float64)
        rhs = np.zeros(6 * n, np.float64)
        fr = np.zeros(n, np.int32)
        x = np.zeros(6 * n, np.float64)
        _lib().oracle_go_first_system(self._h, len(edges), ei.ctypes.data, ej.ctypes.data, iters, H.ctypes.data, rhs.ctypes.data,
                                      fr.ctypes.data, x.ctypes.data)
        return H, rhs, fr.astype(bool), x


def ate(est, gt):
    """(RMS translation error in metres, largest rotation error in degrees) over the poses"""
    te, re = [], []
    for E, G in zip(est, gt):
        te.append(np.linalg.norm(E[:3, 3].astype(np.float64) - G[:3, 3]))
        Rr = E[:3, :3].astype(np.float64).T @ G[:3, :3].astype(np.float64)
        re.append(np.degrees(np.arccos(np.clip((np.trace(Rr) - 1) / 2, -1, 1))))
    return float(np.sqrt(np.mean(np.square(te)))), float(np.max(re))


def scene(W, H, seed=2, size=(5.0, 4.0, 3.0)):
    from scannet_b200 import synth
    return synth.BoxRoomScene(size=size, n_spheres=10, seed=seed, width=W, height=H, fx=synth.FX * W / 640, fy=synth.FY * H / 480,
                              cx=(W - 1) / 2, cy=(H - 1) / 2)


def drift(s, rot_deg, trans):
    """the drift at fraction s of the loop: a rotation of s * rot_deg about the vertical axis through the room centre (2.5, 2, 0)
    and a translation s * trans, applied on the left of a cam2world pose"""
    a = np.radians(rot_deg * s)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    c = np.array([2.5, 2.0, 0.0])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = c - R @ c + s * np.asarray(trans, np.float64)
    return T


def loop_keyframes(sc, n, rot_deg=2.0, trans=(0.03, -0.02, 0.01), noise_mm=1.0, bad=None, bad_seed=7):
    """n keyframes around the closed orbit rendered at the true poses; initial poses carry a drift that grows along the loop.
    Keyframe `bad` (if any) is rendered from another scene (another seed's spheres in a larger room) through one of its outward
    views, so that nothing in it lines up with its neighbours.  Returns depth, true poses, drifted poses."""
    D = np.zeros((n, sc.H, sc.W), np.uint16)
    P = np.zeros((n, 4, 4), np.float32)
    Q = np.zeros((n, 4, 4), np.float32)
    other = scene(sc.W, sc.H, bad_seed, size=(5.8, 4.6, 3.4)) if bad is not None else None
    for k in range(n):
        P[k] = sc.orbit_pose(k, n, height=2.2)
        D[k] = sc.render(P[k], noise_mm=noise_mm, frame_seed=k)[0] if k != bad else \
            other.render(other.camera_pose(3, 12), noise_mm=noise_mm, frame_seed=k)[0]
        Q[k] = (drift(k / (n - 1), rot_deg, trans) @ P[k].astype(np.float64)).astype(np.float32)
    return D, P, Q
