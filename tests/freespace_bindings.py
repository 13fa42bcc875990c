"""ctypes bindings for the free-space oracle (oracle/_build/liboracle_freespace.so, DESIGN.md §6h), plus the spec's label, crop
and .grid steps restated in numpy.  TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and scripts/bench_freespace.py
import this."""
from __future__ import annotations

import ctypes as C
import os
import struct

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle/_build/liboracle_freespace.so")

_o = None


def _lib():
    global _o
    if _o is None:
        if not os.path.exists(ORACLE):
            raise FileNotFoundError(f"{ORACLE} missing — run `make oracle` (oracle/freespace.mk)")
        _o = C.CDLL(ORACLE)
        _o.oracle_freespace_integrate.restype = C.c_uint32
        _o.oracle_freespace_integrate.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.c_void_p, C.c_void_p, C.c_uint32,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    return _o


class OracleCounts:
    """Dense counts over the box lo .. lo+dims-1 (dims = (x, y, z); arrays [z, y, x]), accumulated frame by frame."""

    def __init__(self, params, lo, dims, width, height, depth_shift=1000.0, threads=None):
        self.p, self.W, self.H, self.shift = params, int(width), int(height), float(depth_shift)
        self.lo = np.ascontiguousarray(lo, np.int32); self.dims = np.ascontiguousarray(dims, np.uint64)
        shape = tuple(int(x) for x in self.dims[::-1])
        self.n_free = np.zeros(shape, np.uint32); self.n_occ = np.zeros(shape, np.uint32)
        self.threads = threads or min(32, os.cpu_count() or 1)
        self.frames_used = 0

    def integrate(self, depth, poses, K):
        D = np.ascontiguousarray(depth, np.uint16).reshape(-1, self.H * self.W)
        P = np.ascontiguousarray(poses, np.float32).reshape(-1, 16); Kf = np.ascontiguousarray(K, np.float32).reshape(16)
        self.frames_used += _lib().oracle_freespace_integrate(C.byref(self.p), self.W, self.H, self.shift, self.lo.ctypes.data, self.dims.ctypes.data,
                                                              len(P), D.ctypes.data, P.ctypes.data, Kf.ctypes.data, self.n_free.ctypes.data,
                                                              self.n_occ.ctypes.data, self.threads)
        return self

    def result(self):
        return crop(self.lo, self.n_free, self.n_occ)


def labels_of(n_free, n_occ):
    """spec step D: 0 unknown, 1 free, 2 occupied"""
    lab = np.where((n_free | n_occ) == 0, 0, np.where((n_occ > 0) & (n_occ >= n_free), 2, 1))
    return lab.astype(np.uint8)


def crop(lo, n_free, n_occ):
    """spec step E: (lo, dims (x,y,z), labels, n_free, n_occ) of the smallest box holding every labelled voxel"""
    lab = labels_of(n_free, n_occ)
    nz = np.nonzero(lab)
    if len(nz[0]) == 0:
        e = np.zeros((0, 0, 0), np.uint8)
        return np.zeros(3, np.int32), (0, 0, 0), e, e.astype(np.uint32), e.astype(np.uint32)
    a = [int(x.min()) for x in nz]; b = [int(x.max()) + 1 for x in nz]                 # z, y, x
    s = tuple(slice(a[i], b[i]) for i in range(3))
    olo = np.asarray([lo[0] + a[2], lo[1] + a[1], lo[2] + a[0]], np.int32)
    return olo, (b[2] - a[2], b[1] - a[1], b[0] - a[0]), lab[s].copy(), n_free[s].copy(), n_occ[s].copy()


def grid_bytes(voxel_size, lo, dims, labels):
    """the .grid file of DESIGN.md §6h, written independently of the library"""
    return (b"SCNGRID\0" + struct.pack("<If", 1, voxel_size) + struct.pack("<QQQ", *[int(x) for x in dims]) +
            struct.pack("<iii", *[int(x) for x in lo]) + np.ascontiguousarray(labels, np.uint8).tobytes())


def oracle_grid(params, lo, dims, width, height, depth, poses, K, depth_shift=1000.0):
    """(lo, dims, labels, n_free, n_occ) of the oracle over the box lo/dims"""
    return OracleCounts(params, lo, dims, width, height, depth_shift).integrate(depth, poses, K).result()
