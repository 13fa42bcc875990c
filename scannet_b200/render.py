"""Host-side mirror of the render stage (``scn_render_*``, DESIGN.md §6i): path-traced preview images of a mesh, standing in
for /root/reference/Server/mts_render.py (``<id>_vh_clean_2.ply`` -> ``<id>_vh_clean_2.png``).  The image is this
repository's "render spec v1", not Mitsuba's.  All compute happens in libscannet_b200.so (CUDA)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib

PATH = 0
AO = 1


class RenderParams(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("samples", C.c_uint32), ("integrator", C.c_int32),
                ("max_depth", C.c_uint32), ("exposure", C.c_float), ("world_up", C.c_float * 3), ("camera_up", C.c_float * 3),
                ("camera_offset", C.c_float * 3), ("bsphere_mult", C.c_float)]


class RenderCamera(C.Structure):
    _fields_ = [("origin", C.c_float * 3), ("p00", C.c_float * 3), ("du", C.c_float * 3), ("dv", C.c_float * 3),
                ("t_near", C.c_float), ("t_eps", C.c_float), ("ao_length", C.c_float)]

    def as_array(self) -> np.ndarray:
        """The 15 binary32 values in struct order (origin, p00, du, dv, t_near, t_eps, ao_length)."""
        return np.frombuffer(bytes(self), np.float32).copy()


class RenderReport(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ("views", "pixels", "samples", "primary_rays", "secondary_rays", "primary_hits",
                                          "node_visits", "triangle_tests", "bvh_nodes")] + \
              [(k, C.c_double) for k in ("upload_ms", "bvh_ms", "trace_ms", "download_ms", "total_ms")]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


COUNTERS = ["primary_rays", "secondary_rays", "primary_hits"]     # the counters the oracle reproduces


def default_params(**over) -> RenderParams:
    p = RenderParams()
    lib().scn_render_default_params(C.byref(p))
    for k, v in over.items():
        if k == "integrator" and isinstance(v, str):
            v = {"path": PATH, "ao": AO}[v]
        if k in ("world_up", "camera_up", "camera_offset"):
            v = (C.c_float * 3)(*v)
        setattr(p, k, v)
    return p


def camera(xyz: np.ndarray, params: RenderParams | None = None, theta: float = 0.0, turntable: bool = False) -> RenderCamera:
    """scn_render_camera: the binary32 camera of one view."""
    p = params if params is not None else default_params()
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    cam = RenderCamera()
    lib().scn_render_camera.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_double, C.c_int, C.c_void_p]
    check(lib().scn_render_camera(xyz.ctypes.data, len(xyz), C.byref(p), float(theta), int(bool(turntable)), C.byref(cam)))
    return cam


def turntable_angles(frames_per_degree: int = 5) -> list:
    """The script's turntable: floor(360 / D) views at i * D degrees (D is degrees per frame despite its name)."""
    return [i * frames_per_degree for i in range(360 // frames_per_degree)]


def turntable_names(mesh: str, frames_per_degree: int = 5) -> list:
    return ["{0}_%03i.png".format(mesh) % i for i in range(360 // frames_per_degree)]


def render(xyz: np.ndarray, rgb: np.ndarray | None, tri: np.ndarray, params: RenderParams | None = None, cams=None):
    """Returns (rgba uint8[n_views, H, W, 4], report dict).  cams: one RenderCamera or a list (default: the single view)."""
    p = params if params is not None else default_params()
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3); tri = np.ascontiguousarray(tri, np.uint32).reshape(-1, 3)
    if rgb is not None:
        rgb = np.ascontiguousarray(rgb, np.uint8).reshape(-1, 3)
    if cams is None:
        cams = [camera(xyz, p)]
    elif isinstance(cams, RenderCamera):
        cams = [cams]
    arr = (RenderCamera * len(cams))(*cams)
    out = np.zeros((len(cams), p.height, p.width, 4), np.uint8)
    rep = RenderReport()
    check(lib().scn_render_mesh(xyz.ctypes.data_as(C.c_void_p), rgb.ctypes.data_as(C.c_void_p) if rgb is not None else None,
                                C.c_uint64(len(xyz)), tri.ctypes.data_as(C.c_void_p), C.c_uint64(len(tri)), C.byref(p), arr,
                                C.c_uint32(len(cams)), out.ctypes.data_as(C.c_void_p), C.byref(rep)))
    return out, rep.as_dict()


def main(argv: list) -> int:
    """scn_render_main with argv[1:] = argv (the `render` CLI in-process)."""
    args = [b"render"] + [str(a).encode() for a in argv]
    arr = (C.c_char_p * len(args))(*args)
    return lib().scn_render_main(len(args), arr)


def report_sizeof() -> int:
    lib().scn_render_report_sizeof.restype = C.c_size_t
    return lib().scn_render_report_sizeof()
