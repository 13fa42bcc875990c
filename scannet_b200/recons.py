"""Camera tracking of the `recons` stage (DESIGN.md §6j): thin ctypes mirror of ``scn_track_*``.

A frame-to-model point-to-plane ICP against a raycast of the TSDF volume, each frame integrated at its tracked pose: the tracker
the reference pipeline gets from FriedLiver.exe (BundleFusion), restated as this repository's own spec.  It is NOT BundleFusion's
trajectory: no sparse features, no global optimisation, no relocalisation."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib
from .tsdf import TsdfVolume

LEVELS = 3


class TrackParams(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("dist_thresh", C.c_float), ("normal_thresh", C.c_float),
                ("ray_increment_factor", C.c_float)]


class TrackFrame(C.Structure):
    _fields_ = [("cam2world", C.c_float * 16), ("iterations", C.c_uint32 * LEVELS), ("pairs", C.c_uint32),
                ("valid_pixels", C.c_uint32), ("lost", C.c_uint32), ("residual_ss", C.c_double), ("rms", C.c_double)]


def default_params(**over) -> TrackParams:
    p = TrackParams()
    lib().scn_track_default_params(C.byref(p))
    for k, v in over.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def params_from_file(path: str, base: TrackParams | None = None) -> TrackParams:
    p = base or default_params()
    check(lib().scn_track_params_from_file(path.encode(), C.byref(p)))
    return p


def frame_dict(f: TrackFrame) -> dict:
    return dict(cam2world=np.ctypeslib.as_array(f.cam2world).reshape(4, 4).copy(), iterations=tuple(f.iterations), pairs=f.pairs,
                valid_pixels=f.valid_pixels, lost=f.lost, residual_ss=f.residual_ss, rms=f.rms)


class Tracker:
    """Tracks frames into `volume` (a TsdfVolume).  frames_device(): depth / colour already in device memory (data pointers, e.g.
    torch tensors'); frames(): host arrays, uploaded first."""

    def __init__(self, volume: TsdfVolume, params: TrackParams | None = None):
        self.volume = volume
        self.params = params or default_params()
        self._h = C.c_void_p()
        check(lib().scn_track_create(volume._h, C.byref(self.params), C.byref(self._h)))

    def close(self):
        if self._h:
            lib().scn_track_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def frames_device(self, n: int, d_depth: int, d_rgb: int | None, K, first_pose=None) -> list[dict]:
        Kc = np.ascontiguousarray(K, np.float32)
        P = np.ascontiguousarray(np.eye(4, dtype=np.float32) if first_pose is None else first_pose, np.float32)
        out = (TrackFrame * max(n, 1))()
        check(lib().scn_track_frames(self._h, C.c_uint32(n), C.c_void_p(d_depth), C.c_void_p(d_rgb) if d_rgb else None,
                                     Kc.ctypes.data_as(C.c_void_p), P.ctypes.data_as(C.c_void_p), out))
        return [frame_dict(out[i]) for i in range(n)]

    def frames(self, depth: np.ndarray, rgb, K, first_pose=None) -> list[dict]:
        depth = np.ascontiguousarray(depth, np.uint16)
        L = lib()
        dd = L.scn_device_alloc(depth.nbytes)
        dc = None
        try:
            check(L.scn_memcpy_h2d(dd, depth.ctypes.data, depth.nbytes, None))
            if rgb is not None:
                rgb = np.ascontiguousarray(rgb, np.uint8)
                dc = L.scn_device_alloc(rgb.nbytes)
                check(L.scn_memcpy_h2d(dc, rgb.ctypes.data, rgb.nbytes, None))
            return self.frames_device(len(depth), dd, dc, K, first_pose)
        finally:
            L.scn_device_free(dd)
            if dc:
                L.scn_device_free(dc)

    def stats(self) -> dict:
        f, n = C.c_uint64(0), C.c_uint64(0)
        check(lib().scn_track_stats(self._h, C.byref(f), C.byref(n)))
        return dict(frames=f.value, kernel_launches=n.value)


class ReconsReport(C.Structure):
    """= scn_recons_report_t"""
    _fields_ = [("status", C.c_int32), ("device", C.c_int32)] + [(k, C.c_uint64) for k in (
        "frames", "frames_tracked", "frames_lost", "blocks_allocated", "mesh_vertices", "mesh_faces", "kernel_launches")] + [
        (k, C.c_double) for k in ("setup_s", "recons_s", "decode_s", "track_s", "filter_pyramid_ms", "icp_ms", "integrate_ms", "raycast_ms",
                                  "mc_s", "ply_s", "sens_s", "total_s")]


def recons_scene(sens_path: str, out_ply: str | None, out_sens: str | None = None, params=None, track_params: TrackParams | None = None,
                 device: int = 0) -> dict:
    """The `recons` stage (scn_recons_scene): .sens -> tracked + fused volume -> out_ply, trajectory -> out_sens (None: in place)."""
    from .tsdf import default_params as tsdf_defaults
    p = params or tsdf_defaults(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02)
    tp = track_params or default_params()
    r = ReconsReport()
    check(lib().scn_recons_scene(sens_path.encode(), out_ply.encode() if out_ply else None, out_sens.encode() if out_sens else None,
                                 C.byref(p), C.byref(tp), device, C.byref(r)))
    return {k: getattr(r, k) for k, _ in ReconsReport._fields_}


def phase_ms(tracker: Tracker) -> dict:
    v = [C.c_double(0) for _ in range(4)]
    check(lib().scn_track_phase_ms(tracker._h, *[C.byref(x) for x in v]))
    return dict(zip(("frame_maps", "icp", "integrate", "raycast"), (x.value for x in v)))


# ---------------------------------------------------------------------------------------------------------------------------------
# Global optimisation of the keyframe trajectory (DESIGN.md §6k): ctypes mirror of ``scn_globalopt_*``.

MAX_NONLIN = 16


class GlobalParams(C.Structure):
    """= scn_globalopt_params"""
    _fields_ = [("submap_size", C.c_uint32), ("max_keyframes", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32),
                ("dist_thresh", C.c_float), ("normal_thresh", C.c_float), ("depth_min", C.c_float), ("depth_max", C.c_float),
                ("overlap_subsample", C.c_uint32), ("nonlin_iters", C.c_uint32), ("lin_iters", C.c_uint32), ("verify_thresh", C.c_float),
                ("max_removed", C.c_uint32)]


class GlobalReport(C.Structure):
    """= scn_globalopt_report_t"""
    _fields_ = [(k, C.c_uint32) for k in ("keyframes", "edges_consecutive", "edges_loop", "edges_removed", "rejected", "solves",
                                          "nonlin_iterations", "lin_iterations")] + [
        ("pairs_before", C.c_uint64), ("pairs_after", C.c_uint64)] + [
        (k, C.c_double) for k in ("rss_before", "rss_after", "rms_before", "rms_after", "max_edge_rms")] + [
        ("rss_iter", C.c_double * MAX_NONLIN)] + [
        (k, C.c_double) for k in ("keyframe_maps_ms", "overlap_ms", "linearise_ms", "pcg_ms", "verify_ms")]


class GlobalEdge(C.Structure):
    """= scn_globalopt_edge_t"""
    _fields_ = [(k, C.c_uint32) for k in ("i", "j", "loop", "removed", "pairs", "pad_")] + [("rss", C.c_double), ("rms", C.c_double)]


def global_default_params(**over) -> GlobalParams:
    p = GlobalParams()
    lib().scn_globalopt_default_params(C.byref(p))
    for k, v in over.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def global_params_from_file(path: str, base: GlobalParams | None = None) -> GlobalParams:
    p = base or global_default_params()
    check(lib().scn_globalopt_params_from_file(path.encode(), C.byref(p)))
    return p


def report_dict(r: GlobalReport) -> dict:
    d = {k: getattr(r, k) for k, _ in GlobalReport._fields_ if k != "rss_iter"}
    d["rss_iter"] = tuple(r.rss_iter)
    return d


def keyframe_indices(lost, submap_size: int) -> list[int]:
    """The keyframe of each submap of `submap_size` consecutive frames: its first frame that was tracked (lost[f] == 0); a submap
    whose frames are all lost has none."""
    out = []
    for s in range(0, len(lost), submap_size):
        for f in range(s, min(s + submap_size, len(lost))):
            if not lost[f]:
                out.append(f)
                break
    return out


class GlobalOptimizer:
    """Keyframes of one trajectory and their global optimisation, bound to `volume` (a TsdfVolume: depth resolution, depth shift,
    filter and stream).  add_keyframes_device(): depth in device memory (data pointers, e.g. torch tensors'); add_keyframes(): host
    arrays or CUDA torch tensors."""

    def __init__(self, volume: TsdfVolume, params: GlobalParams | None = None):
        self.volume = volume
        self.params = params or global_default_params()
        self._h = C.c_void_p()
        self.n = 0
        check(lib().scn_globalopt_create(volume._h, C.byref(self.params), C.byref(self._h)))

    def close(self):
        if self._h:
            lib().scn_globalopt_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def add_keyframes_device(self, n: int, d_depth: int, poses, K):
        P = np.ascontiguousarray(np.asarray(poses, np.float32).reshape(-1, 16)[:n])
        Kc = np.ascontiguousarray(K, np.float32)
        check(lib().scn_globalopt_add_keyframes(self._h, C.c_uint32(n), C.c_void_p(d_depth), P.ctypes.data_as(C.c_void_p),
                                                Kc.ctypes.data_as(C.c_void_p)))
        self.n += n

    def add_keyframes(self, depth, poses, K):
        if hasattr(depth, "is_cuda") and depth.is_cuda:
            return self.add_keyframes_device(int(depth.shape[0]), depth.data_ptr(), poses, K)
        depth = np.ascontiguousarray(depth, np.uint16)
        L = lib()
        dd = L.scn_device_alloc(max(depth.nbytes, 1))
        try:
            check(L.scn_memcpy_h2d(dd, depth.ctypes.data, depth.nbytes, None))
            self.add_keyframes_device(len(depth), dd, poses, K)
        finally:
            L.scn_device_free(dd)

    def solve(self):
        """(poses (keyframes, 4, 4) float32, report dict)"""
        out = np.zeros((max(self.n, 1), 4, 4), np.float32)
        r = GlobalReport()
        check(lib().scn_globalopt_solve(self._h, out.ctypes.data_as(C.c_void_p), C.byref(r)))
        return out[:self.n], report_dict(r)

    def edges(self) -> list[dict]:
        n = C.c_uint32(0)
        check(lib().scn_globalopt_edges(self._h, None, 0, C.byref(n)))
        buf = (GlobalEdge * max(n.value, 1))()
        check(lib().scn_globalopt_edges(self._h, buf, n.value, C.byref(n)))
        return [{k: getattr(buf[e], k) for k, _ in GlobalEdge._fields_ if k != "pad_"} for e in range(n.value)]


def recons_scene_global(sens_path: str, out_ply: str | None, out_sens: str | None = None, params=None,
                        track_params: TrackParams | None = None, global_params: GlobalParams | None = None, device: int = 0):
    """`recons --global` (scn_recons_scene_global): the `recons` stage with the keyframe trajectory optimised, propagated to every
    tracked frame and the stream re-integrated at the new poses.  Returns (recons report dict, global report dict)."""
    from .tsdf import default_params as tsdf_defaults
    p = params or tsdf_defaults(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02)
    tp = track_params or default_params()
    gp = global_params or global_default_params()
    r, g = ReconsReport(), GlobalReport()
    check(lib().scn_recons_scene_global(sens_path.encode(), out_ply.encode() if out_ply else None, out_sens.encode() if out_sens else None,
                                        C.byref(p), C.byref(tp), C.byref(gp), device, C.byref(r), C.byref(g)))
    return {k: getattr(r, k) for k, _ in ReconsReport._fields_}, report_dict(g)


def propagate(Tk, Tk_new, Tf):
    """T_f' = T_k' (T_k^-1 T_f) in binary64 in the library's order, rounded once (scn_recons_scene_global's propagation)."""
    a, b, f = (np.asarray(x, np.float32).astype(np.float64) for x in (Tk, Tk_new, Tf))
    A = np.zeros((3, 4))
    for r in range(3):
        for c in range(4):
            m = (a[0, r] * f[0, c] + a[1, r] * f[1, c]) + a[2, r] * f[2, c]
            if c == 3:
                m = m - ((a[0, r] * a[0, 3] + a[1, r] * a[1, 3]) + a[2, r] * a[2, 3])
            A[r, c] = m
    out = np.eye(4, dtype=np.float32)
    for r in range(3):
        for c in range(4):
            m = (b[r, 0] * A[0, c] + b[r, 1] * A[1, c]) + b[r, 2] * A[2, c]
            if c == 3:
                m = m + b[r, 3]
            out[r, c] = np.float32(m)
    return out
