"""ctypes bindings for the tracker oracle (oracle/_build/liboracle_track.so, DESIGN.md §6j).  TEST INFRASTRUCTURE: only tests/,
__graft_entry__.smoke() and scripts/bench_recons.py import this."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle_bindings import VOXEL_DTYPE, OracleTsdfParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle/_build/liboracle_track.so")
NSUM = 28
LEVELS = 3


class OracleTrackParams(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("dist_thresh", C.c_float), ("normal_thresh", C.c_float),
                ("ray_increment_factor", C.c_float)]


class TrackFrame(C.Structure):
    """= scn_track_frame_t"""
    _fields_ = [("cam2world", C.c_float * 16), ("iterations", C.c_uint32 * LEVELS), ("pairs", C.c_uint32),
                ("valid_pixels", C.c_uint32), ("lost", C.c_uint32), ("residual_ss", C.c_double), ("rms", C.c_double)]


def frame_dict(f: TrackFrame) -> dict:
    return dict(cam2world=np.ctypeslib.as_array(f.cam2world).reshape(4, 4).copy(), iterations=tuple(f.iterations), pairs=f.pairs,
                valid_pixels=f.valid_pixels, lost=f.lost, residual_ss=f.residual_ss, rms=f.rms)


_o = None


def _lib():
    global _o
    if _o is None:
        if not os.path.exists(ORACLE):
            raise FileNotFoundError(f"{ORACLE} missing — run `make oracle` (oracle/track.mk)")
        _o = C.CDLL(ORACLE)
        _o.oracle_track_create.restype = C.c_void_p
        _o.oracle_track_create.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        _o.oracle_track_destroy.argtypes = [C.c_void_p]
        _o.oracle_track_volume.restype = C.c_void_p
        _o.oracle_track_volume.argtypes = [C.c_void_p]
        _o.oracle_track_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _o.oracle_track_set_frame.restype = C.c_uint32
        _o.oracle_track_set_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _o.oracle_track_system.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _o.oracle_track_terms.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _o.oracle_track_maps.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4
        _o.oracle_track_model_depth.argtypes = [C.c_void_p, C.c_void_p]
        _o.oracle_track_solve.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        _o.oracle_track_cayley.argtypes = [C.c_void_p, C.c_void_p]
        _o.oracle_tsdf_num_blocks.restype = C.c_uint64
        _o.oracle_tsdf_num_blocks.argtypes = [C.c_void_p]
        _o.oracle_tsdf_export.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _o.oracle_tsdf_extract_mesh.argtypes = [C.c_void_p, C.c_float] + [C.c_void_p] * 5
        _o.oracle_free.argtypes = [C.c_void_p]
    return _o


def metres(depth_u16, depth_shift=1000.0):
    """Unfiltered metres as the tracker reads them: raw / depth_shift, -inf where raw == 0."""
    d = np.asarray(depth_u16)
    m = d.astype(np.float32) / np.float32(depth_shift)
    return np.where(d == 0, np.float32(-np.inf), m).astype(np.float32)


def cayley(w):
    R = np.zeros(9, np.float64)
    _lib().oracle_track_cayley(np.ascontiguousarray(w, np.float64).ctypes.data, R.ctypes.data)
    return R.reshape(3, 3)


def solve(sums, pairs):
    """Cholesky solve of the 28 sums (JtJ upper triangle row-major, Jtr, sum r^2): x or None when not positive definite."""
    x = np.zeros(6, np.float64)
    ok = _lib().oracle_track_solve(np.ascontiguousarray(sums, np.float64).ctypes.data, pairs, x.ctypes.data)
    return x if ok else None


class OracleTracker:
    """Tracker + volume of the oracle.  vparams: an object with the scn_tsdf_params fields of OracleTsdfParams; tparams: one with
    width, height, dist_thresh, normal_thresh, ray_increment_factor."""

    def __init__(self, vparams, tparams, threads: int = 0):
        vp = OracleTsdfParams()
        for f, _ in OracleTsdfParams._fields_:
            setattr(vp, f, getattr(vparams, f))
        tp = OracleTrackParams()
        for f, _ in OracleTrackParams._fields_:
            setattr(tp, f, getattr(tparams, f))
        self._vp, self._tp = vp, tp
        self.W, self.H = int(vp.width), int(vp.height)
        self._h = _lib().oracle_track_create(C.byref(vp), C.byref(tp), threads or os.cpu_count() or 1)
        if not self._h:
            raise ValueError("tracking resolution is not the depth resolution divided by a power of two")

    def __del__(self):
        if getattr(self, "_h", None):
            _lib().oracle_track_destroy(self._h)
            self._h = None

    def frame(self, metres_img, rgb, K, first_pose=None) -> dict:
        m = np.ascontiguousarray(metres_img, np.float32)
        assert m.shape == (self.H, self.W)
        Kc = np.ascontiguousarray(K, np.float32)
        P = np.ascontiguousarray(np.eye(4, dtype=np.float32) if first_pose is None else first_pose, np.float32)
        rp = None
        if rgb is not None:
            rgb = np.ascontiguousarray(rgb, np.uint8); rp = rgb.ctypes.data
        out = TrackFrame()
        _lib().oracle_track_frame(self._h, m.ctypes.data, rp, Kc.ctypes.data, P.ctypes.data, C.byref(out))
        return frame_dict(out)

    def set_frame(self, metres_img, K) -> int:
        m = np.ascontiguousarray(metres_img, np.float32); Kc = np.ascontiguousarray(K, np.float32)
        return int(_lib().oracle_track_set_frame(self._h, m.ctypes.data, Kc.ctypes.data))

    def level_size(self, k):
        return int(self._tp.width) >> k, int(self._tp.height) >> k

    def system(self, k, D):
        Df = np.ascontiguousarray(np.asarray(D, np.float32)[:3, :4])
        s = np.zeros(NSUM, np.float64); n = C.c_uint32(0)
        _lib().oracle_track_system(self._h, k, Df.ctypes.data, s.ctypes.data, C.byref(n))
        return s, int(n.value)

    def terms(self, k, D):
        w, h = self.level_size(k)
        Df = np.ascontiguousarray(np.asarray(D, np.float32)[:3, :4])
        t = np.zeros((w * h, NSUM), np.float64); p = np.zeros(w * h, np.uint8)
        _lib().oracle_track_terms(self._h, k, Df.ctypes.data, t.ctypes.data, p.ctypes.data)
        return t, p

    def maps(self, k):
        w, h = self.level_size(k)
        a = [np.zeros((h, w, 4), np.float32) for _ in range(4)]
        _lib().oracle_track_maps(self._h, k, *[x.ctypes.data for x in a])
        return a

    def model_depth(self):
        w, h = self.level_size(0)
        d = np.zeros((h, w), np.float32)
        _lib().oracle_track_model_depth(self._h, d.ctypes.data)
        return d

    def export(self):
        v = _lib().oracle_track_volume(self._h)
        n = _lib().oracle_tsdf_num_blocks(v)
        xyz = np.zeros((n, 3), np.int32); vox = np.zeros((n, 512), VOXEL_DTYPE)
        if n:
            _lib().oracle_tsdf_export(v, xyz.ctypes.data, vox.ctypes.data)
        return xyz, vox

    def extract_mesh(self, thresh_factor=10.0):
        v = _lib().oracle_track_volume(self._h)
        px, pc, pt = C.c_void_p(), C.c_void_p(), C.c_void_p(); nv, nf = C.c_uint64(0), C.c_uint64(0)
        _lib().oracle_tsdf_extract_mesh(v, thresh_factor, C.byref(px), C.byref(pc), C.byref(pt), C.byref(nv), C.byref(nf))
        xyz = np.ctypeslib.as_array((C.c_float * (3 * nv.value)).from_address(px.value)).reshape(-1, 3).copy() if nv.value else np.zeros((0, 3), np.float32)
        rgb = np.ctypeslib.as_array((C.c_uint8 * (3 * nv.value)).from_address(pc.value)).reshape(-1, 3).copy() if nv.value else np.zeros((0, 3), np.uint8)
        tri = np.ctypeslib.as_array((C.c_uint32 * (3 * nf.value)).from_address(pt.value)).reshape(-1, 3).copy() if nf.value else np.zeros((0, 3), np.uint32)
        for p in (px, pc, pt):
            _lib().oracle_free(p)
        return xyz, rgb, tri


def pose_errors(est, gt):
    """(translation RMS over the tracked frames, max rotation error in degrees); frames with an invalid estimate are skipped."""
    te, re = [], []
    for E, G in zip(est, gt):
        if not np.isfinite(E).all():
            continue
        te.append(np.linalg.norm(E[:3, 3].astype(np.float64) - G[:3, 3]))
        Rr = E[:3, :3].astype(np.float64).T @ G[:3, :3].astype(np.float64)
        re.append(np.degrees(np.arccos(np.clip((np.trace(Rr) - 1) / 2, -1, 1))))
    return float(np.sqrt(np.mean(np.square(te)))), float(np.max(re))
