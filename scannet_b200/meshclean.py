"""Host-side mirror of the mesh-cleaning stage (``scn_mesh_clean``, DESIGN.md §6f): MeshLab's clean.mlx step of the ScanNet
``decimate`` stage (/root/reference/Server/scan_processor.py:143, ``<id>_vh.ply`` -> ``<id>_vh_clean.ply``) stated as mLib's
MeshData operators.  All compute happens in libscannet_b200.so (CUDA)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib

SKIP_MERGE = 1
SKIP_DEDUP = 2
SKIP_PIECES = 4


class CleanParams(C.Structure):
    _fields_ = [("merge_threshold", C.c_float), ("min_piece_vertices", C.c_uint32), ("min_piece_faces", C.c_uint32), ("flags", C.c_uint32)]


class CleanReport(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ("vertices_in", "faces_in", "vertices_out", "faces_out", "vertices_merged", "merge_components",
                                          "largest_merge_component", "degenerate_faces", "duplicate_faces", "pieces_total", "pieces_removed",
                                          "faces_in_removed_pieces")] + \
              [(k, C.c_double) for k in ("upload_ms", "merge_ms", "dedup_ms", "pieces_ms", "download_ms", "total_ms")]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


COUNTERS = [k for k, t in CleanReport._fields_ if t is C.c_uint64][4:]     # the fields the CPU oracle reproduces, in its order


def default_params(**over) -> CleanParams:
    p = CleanParams()
    lib().scn_mesh_clean_default_params(C.byref(p))
    for k, v in over.items():
        setattr(p, k, v)
    return p


def params_from_mlx(path: str, base: CleanParams | None = None) -> CleanParams:
    p = base if base is not None else default_params()
    check(lib().scn_mesh_clean_params_from_mlx(str(path).encode(), C.byref(p)))
    return p


def _take(ptr, n, dtype, cols):
    if not ptr:
        return None
    ct = {np.float32: C.c_float, np.uint8: C.c_uint8, np.uint32: C.c_uint32}[dtype]
    a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), (max(int(n) * cols, 1),))[: int(n) * cols].copy().reshape(-1, cols)
    lib().scn_free(C.cast(ptr, C.c_void_p))
    return a


def clean(xyz: np.ndarray, tri: np.ndarray, rgb: np.ndarray | None = None, params: CleanParams | None = None, **over):
    """Returns (xyz float32[V,3], rgb uint8[V,3] or None, tri uint32[F,3], report dict)."""
    p = params if params is not None else default_params()
    for k, v in over.items():
        setattr(p, k, v)
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3); tri = np.ascontiguousarray(tri, np.uint32).reshape(-1, 3)
    if rgb is not None:
        rgb = np.ascontiguousarray(rgb, np.uint8).reshape(-1, 3)
    ox = C.POINTER(C.c_float)(); oc = C.POINTER(C.c_uint8)(); ot = C.POINTER(C.c_uint32)(); nv = C.c_uint64(); nf = C.c_uint64()
    rep = CleanReport()
    check(lib().scn_mesh_clean(xyz.ctypes.data_as(C.c_void_p), rgb.ctypes.data_as(C.c_void_p) if rgb is not None else None, C.c_uint64(len(xyz)),
                               tri.ctypes.data_as(C.c_void_p), C.c_uint64(len(tri)), C.byref(p), C.byref(ox), C.byref(oc), C.byref(ot),
                               C.byref(nv), C.byref(nf), C.byref(rep)))
    x = _take(ox, nv.value, np.float32, 3); c = _take(oc, nv.value, np.uint8, 3); t = _take(ot, nf.value, np.uint32, 3)
    return x, c, t, rep.as_dict()


def load_rgb(path: str):
    """scn_mesh_load_rgb: (xyz float32[V,3], rgb uint8[V,3] or None, tri uint32[F,3])."""
    x = C.POINTER(C.c_float)(); c = C.POINTER(C.c_uint8)(); t = C.POINTER(C.c_uint32)(); nv = C.c_uint64(); nf = C.c_uint64()
    check(lib().scn_mesh_load_rgb(str(path).encode(), C.byref(x), C.byref(c), C.byref(nv), C.byref(t), C.byref(nf)))
    return _take(x, nv.value, np.float32, 3), _take(c, nv.value, np.uint8, 3), _take(t, nf.value, np.uint32, 3)


def report_sizeof() -> int:
    lib().scn_mesh_clean_report_sizeof.restype = C.c_size_t
    return lib().scn_mesh_clean_report_sizeof()
