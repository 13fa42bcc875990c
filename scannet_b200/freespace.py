"""Host-side mirror of the free-space occupancy grid (``scn_freespace_*``, DESIGN.md §6h): the ScanNet ``freespace`` stage
(Server/scan_processor.py:150-152, ``<id>.sens`` -> ``<id>.grid``) under this repository's own "free-space spec v1".
Labels: 0 unknown, 1 free, 2 occupied.  All compute happens in libscannet_b200.so (CUDA); ``read_grid`` is a plain file reader."""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np

from ._lib import check, lib

GRID_MAGIC = b"SCNGRID\0"
GRID_HEADER = 52


class FreespaceParams(C.Structure):
    _fields_ = [("voxel_size", C.c_float), ("band_base", C.c_float), ("band_scale", C.c_float), ("depth_min", C.c_float),
                ("depth_max", C.c_float), ("max_distance", C.c_float), ("max_voxels", C.c_uint64)]


class FreespaceReport(C.Structure):
    _fields_ = [("frames_used", C.c_uint64), ("frames_skipped_pose", C.c_uint64),
                ("envelope_dims", C.c_uint64 * 3), ("output_dims", C.c_uint64 * 3),
                ("envelope_lo", C.c_int32 * 3), ("output_lo", C.c_int32 * 3)] + \
              [(k, C.c_uint64) for k in ("voxels_free", "voxels_occupied", "voxels_unknown", "pairs_classified", "pairs_culled")] + \
              [(k, C.c_double) for k in ("decode_s", "classify_ms", "crop_ms", "write_s", "total_s")]

    def as_dict(self):
        return {k: (list(getattr(self, k)) if k.endswith(("_dims", "_lo")) else getattr(self, k)) for k, _ in self._fields_}


def default_params(**over) -> FreespaceParams:
    p = FreespaceParams()
    lib().scn_freespace_default_params(C.byref(p))
    for k, v in over.items():
        setattr(p, k, v)
    return p


def _f32(a, shape):
    return np.ascontiguousarray(a, np.float32).reshape(shape)


def envelope(poses, K, width: int, height: int, params: FreespaceParams | None = None):
    """(lo int32[3], dims uint64[3]): the lattice box every observation of frames with these poses falls in (host only)."""
    p = params if params is not None else default_params()
    P = _f32(poses, (-1, 16)); Kf = _f32(K, (16,))
    lo = np.zeros(3, np.int32); dims = np.zeros(3, np.uint64)
    check(lib().scn_freespace_envelope(P.ctypes.data_as(C.c_void_p), C.c_uint32(len(P)), Kf.ctypes.data_as(C.c_void_p), C.c_uint32(width),
                                       C.c_uint32(height), C.byref(p), lo.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p)))
    return lo, dims


def _take(ptr, n, dtype):
    if not ptr:
        return np.zeros(0, dtype)
    a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dtype))), (int(n),)).copy()
    lib().scn_free(C.cast(ptr, C.c_void_p))
    return a


class FreeSpace:
    """Counts over the lattice box lo .. lo+dims-1 for width x height depth frames on one GPU."""

    def __init__(self, lo, dims, width: int, height: int, depth_shift: float = 1000.0, params: FreespaceParams | None = None, device: int = 0):
        self.params = params if params is not None else default_params()
        self._h = C.c_void_p()
        lo = np.ascontiguousarray(lo, np.int32); dims = np.ascontiguousarray(dims, np.uint64)
        check(lib().scn_freespace_create(C.byref(self.params), C.c_uint32(width), C.c_uint32(height), C.c_float(depth_shift),
                                         lo.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p), C.c_int(device), C.byref(self._h)))
        self.W, self.H = width, height

    def integrate(self, depth, poses, K):
        """Host frames: depth uint16 [N,H,W], poses [N,4,4] cam2world (-inf = no pose), K 4x4."""
        D = np.ascontiguousarray(depth, np.uint16).reshape(-1, self.H * self.W)
        P = _f32(poses, (-1, 16)); Kf = _f32(K, (16,))
        assert len(D) == len(P)
        check(lib().scn_freespace_integrate(self._h, C.c_uint32(len(P)), D.ctypes.data_as(C.c_void_p), P.ctypes.data_as(C.c_void_p),
                                            Kf.ctypes.data_as(C.c_void_p)))

    def integrate_device(self, d_depth: int, n: int, poses, K):
        """Frames already in device memory (d_depth: device pointer to n*H*W uint16)."""
        P = _f32(poses, (-1, 16)); Kf = _f32(K, (16,))
        check(lib().scn_freespace_integrate_device(self._h, C.c_uint32(n), C.c_void_p(d_depth), P.ctypes.data_as(C.c_void_p),
                                                   Kf.ctypes.data_as(C.c_void_p)))

    def download(self, counts: bool = True):
        """(lo int32[3], dims (x,y,z), labels uint8 [z,y,x], n_free, n_occ uint32 [z,y,x] or None): the crop box of labelled voxels."""
        lo = np.zeros(3, np.int32); dims = np.zeros(3, np.uint64)
        pl = C.POINTER(C.c_uint8)(); pf = C.POINTER(C.c_uint32)(); po = C.POINTER(C.c_uint32)()
        check(lib().scn_freespace_download(self._h, lo.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p), C.byref(pl),
                                           C.byref(pf) if counts else None, C.byref(po) if counts else None))
        n = int(np.prod(dims))
        shape = tuple(int(x) for x in dims[::-1])
        lab = _take(pl, n, np.uint8).reshape(shape)
        nf = _take(pf, n, np.uint32).reshape(shape) if counts else None
        no = _take(po, n, np.uint32).reshape(shape) if counts else None
        return lo, tuple(int(x) for x in dims), lab, nf, no

    def report(self) -> dict:
        r = FreespaceReport()
        check(lib().scn_freespace_handle_report(self._h, C.byref(r)))
        return r.as_dict()

    def close(self):
        if self._h:
            lib().scn_freespace_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def save_grid(path, voxel_size: float, lo, dims, labels):
    """The library's .grid writer (dims = (x, y, z), labels x fastest)."""
    lo = np.ascontiguousarray(lo, np.int32); dims = np.ascontiguousarray(dims, np.uint64)
    lab = np.ascontiguousarray(labels, np.uint8).reshape(-1)
    check(lib().scn_freespace_save_grid(str(path).encode(), C.c_float(voxel_size), lo.ctypes.data_as(C.c_void_p),
                                        dims.ctypes.data_as(C.c_void_p), lab.ctypes.data_as(C.c_void_p) if lab.size else None))


def read_grid(path):
    """dict(voxel_size, lo (x,y,z), dims (x,y,z), labels uint8 [z,y,x], grid2world 4x4): grid -> world is scale vs, translation vs*lo."""
    with open(path, "rb") as f:
        b = f.read()
    if len(b) < GRID_HEADER or b[:8] != GRID_MAGIC:
        raise ValueError(f"{path}: not a .grid file")
    version, vs = struct.unpack_from("<If", b, 8)
    if version != 1:
        raise ValueError(f"{path}: .grid version {version}")
    dims = struct.unpack_from("<QQQ", b, 16)
    lo = struct.unpack_from("<iii", b, 40)
    n = dims[0] * dims[1] * dims[2]
    if len(b) != GRID_HEADER + n:
        raise ValueError(f"{path}: {len(b) - GRID_HEADER} label bytes, header says {n}")
    labels = np.frombuffer(b, np.uint8, n, GRID_HEADER).reshape(dims[2], dims[1], dims[0])
    g2w = np.eye(4)
    g2w[:3, :3] *= vs
    g2w[:3, 3] = np.asarray(lo, np.float64) * vs
    return {"voxel_size": vs, "lo": lo, "dims": dims, "labels": labels, "grid2world": g2w}


def freespace_scene(sens_path, out_grid=None, params: FreespaceParams | None = None, device: int = 0, **over) -> dict:
    """The stage: .sens -> .grid (out_grid None: no file).  Returns the report as a dict."""
    p = FreespaceParams.from_buffer_copy(params) if params is not None else default_params()     # overrides never touch the caller's struct
    for k, v in over.items():
        setattr(p, k, v)
    r = FreespaceReport()
    check(lib().scn_freespace_scene(str(sens_path).encode(), str(out_grid).encode() if out_grid else None, C.byref(p), C.c_int(device),
                                    C.byref(r)))
    return r.as_dict()


def report_sizeof() -> int:
    lib().scn_freespace_report_sizeof.restype = C.c_size_t
    return lib().scn_freespace_report_sizeof()
