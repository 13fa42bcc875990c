"""Host-side mirror of mesh decimation (``scn_mesh_simplify``, DESIGN.md §6g): MeshLab's simplify.mlx step of the ScanNet
``decimate`` stage (Server/scan_processor.py:144-145, ``<id>_vh_clean.ply`` -> ``_vh_clean_1.ply`` -> ``_vh_clean_2.ply``):
quadric edge collapse in deterministic rounds of independent collapses (this repository's own spec, not MeshLab's output), then
AutoClean and the script's clean filters.  All compute happens in libscannet_b200.so (CUDA)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib
from .meshclean import CleanParams, CleanReport, _take


class SimplifyParams(C.Structure):
    _fields_ = [("target_faces", C.c_uint64), ("target_perc", C.c_double), ("quality_thr", C.c_double)]


class SimplifyReport(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ("vertices_in", "faces_in", "vertices_out", "faces_out", "target_faces", "rounds", "collapses",
                                          "faces_collapsed", "autoclean_duplicate_faces", "max_vertex_faces")] + \
              [(k, C.c_double) for k in ("upload_ms", "quadrics_ms", "rounds_ms", "autoclean_ms", "clean_ms", "download_ms", "total_ms")] + \
              [("clean", CleanReport)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k != "clean"}
        d["clean"] = self.clean.as_dict()
        return d


COUNTERS = [k for k, t in SimplifyReport._fields_ if t is C.c_uint64][4:]    # the fields the CPU oracle reproduces, in its order


def default_params(**over):
    """(SimplifyParams, CleanParams): simplify.mlx's decimation and the clean filters it runs after it."""
    p, a = SimplifyParams(), CleanParams()
    lib().scn_mesh_simplify_default_params(C.byref(p), C.byref(a))
    for k, v in over.items():
        setattr(p, k, v)
    return p, a


def params_from_mlx(path: str):
    """(SimplifyParams, CleanParams) read from a simplify.mlx-shaped FilterScript."""
    p, a = default_params()
    check(lib().scn_mesh_simplify_params_from_mlx(str(path).encode(), C.byref(p), C.byref(a)))
    return p, a


def simplify(xyz: np.ndarray, tri: np.ndarray, rgb: np.ndarray | None = None, params: SimplifyParams | None = None,
             after: CleanParams | None = None, **over):
    """Returns (xyz float32[V,3], rgb uint8[V,3] or None, tri uint32[F,3], report dict).  `after` = None runs no clean filter;
    keyword arguments override fields of `params` (default: simplify.mlx's)."""
    p = params if params is not None else default_params()[0]
    for k, v in over.items():
        setattr(p, k, v)
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3); tri = np.ascontiguousarray(tri, np.uint32).reshape(-1, 3)
    if rgb is not None:
        rgb = np.ascontiguousarray(rgb, np.uint8).reshape(-1, 3)
    ox = C.POINTER(C.c_float)(); oc = C.POINTER(C.c_uint8)(); ot = C.POINTER(C.c_uint32)(); nv = C.c_uint64(); nf = C.c_uint64()
    rep = SimplifyReport()
    check(lib().scn_mesh_simplify(xyz.ctypes.data_as(C.c_void_p), rgb.ctypes.data_as(C.c_void_p) if rgb is not None else None,
                                  C.c_uint64(len(xyz)), tri.ctypes.data_as(C.c_void_p), C.c_uint64(len(tri)), C.byref(p),
                                  C.byref(after) if after is not None else None, C.byref(ox), C.byref(oc), C.byref(ot), C.byref(nv),
                                  C.byref(nf), C.byref(rep)))
    x = _take(ox, nv.value, np.float32, 3); c = _take(oc, nv.value, np.uint8, 3); t = _take(ot, nf.value, np.uint32, 3)
    return x, c, t, rep.as_dict()


def report_sizeof() -> int:
    lib().scn_mesh_simplify_report_sizeof.restype = C.c_size_t
    return lib().scn_mesh_simplify_report_sizeof()
