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
        L.scn_device_alloc.restype = C.c_void_p
        L.scn_device_alloc.argtypes = [C.c_size_t]
        L.scn_device_free.argtypes = [C.c_void_p]
        L.scn_memcpy_h2d.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
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
