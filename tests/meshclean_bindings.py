"""ctypes bindings for the mesh-cleaning oracle (oracle/_build/liboracle_meshclean.so) and the unmodified mLib MeshData operators
(oracle/_ref/libref_meshdata.so).  TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and scripts/bench_meshclean.py import this."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle/_build/liboracle_meshclean.so")
REF = os.path.join(ROOT, "oracle/_ref/libref_meshdata.so")
# counters[] of oracle_mesh_clean, in order (the integer fields of scn_mesh_clean_report_t after the four sizes)
COUNTERS = ["vertices_merged", "merge_components", "largest_merge_component", "degenerate_faces", "duplicate_faces", "pieces_total",
            "pieces_removed", "faces_in_removed_pieces"]
SKIP_MERGE, SKIP_DEDUP, SKIP_PIECES = 1, 2, 4

_o = _r = None


def _lib(path):
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} missing — run `make oracle` (oracle/meshclean.mk)")
    return C.CDLL(path)


def _prep(xyz, tri, rgb):
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3); tri = np.ascontiguousarray(tri, np.uint32).reshape(-1, 3)
    if rgb is not None:
        rgb = np.ascontiguousarray(rgb, np.uint8).reshape(-1, 3)
    return xyz, tri, rgb


class OracleRefusal(ValueError):
    pass


def oracle_clean(xyz, tri, rgb=None, merge_threshold=0.0010689, min_piece_vertices=0, min_piece_faces=7500, flags=0):
    """oracle/meshclean_oracle.c: (xyz, rgb or None, tri, counters dict); raises OracleRefusal where the library gives SCN_ERR_ARG."""
    global _o
    if _o is None:
        _o = _lib(ORACLE)
        _o.oracle_mesh_clean.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_float, C.c_uint32, C.c_uint32,
                                         C.c_uint32] + [C.c_void_p] * 6
    xyz, tri, rgb = _prep(xyz, tri, rgb)
    nV, nF = len(xyz), len(tri)
    ox = np.zeros((max(nV, 1), 3), np.float32); oc = np.zeros((max(nV, 1), 3), np.uint8); ot = np.zeros((max(nF, 1), 3), np.uint32)
    nv = C.c_int64(); nf = C.c_int64(); cnt = np.zeros(len(COUNTERS), np.uint64)
    rc = _o.oracle_mesh_clean(xyz.ctypes.data, rgb.ctypes.data if rgb is not None else None, nV, tri.ctypes.data, nF, merge_threshold,
                              min_piece_vertices, min_piece_faces, flags, ox.ctypes.data, oc.ctypes.data, ot.ctypes.data,
                              C.addressof(nv), C.addressof(nf), cnt.ctypes.data)
    if rc == -1:
        raise OracleRefusal("refused")
    assert rc == 0, rc
    return ox[:nv.value].copy(), (oc[:nv.value].copy() if rgb is not None else None), ot[:nf.value].copy(), dict(zip(COUNTERS, map(int, cnt)))


def have_ref():
    return os.path.exists(REF)


def ref_clean(xyz, tri, rgb=None, merge_threshold=0.0010689, merge=True, dedup=True):
    """mLib MeshData<float>: mergeCloseVertices(t, false) and/or removeDuplicateFaces, unmodified: (xyz, rgb or None, tri)."""
    global _r
    if _r is None:
        _r = _lib(REF)
        _r.ref_mesh_clean.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_float, C.c_int] + [C.c_void_p] * 5
    xyz, tri, rgb = _prep(xyz, tri, rgb)
    nV, nF = len(xyz), len(tri)
    ox = np.zeros((max(nV, 1), 3), np.float32); oc = np.zeros((max(nV, 1), 3), np.uint8); ot = np.zeros((max(nF, 1), 3), np.uint32)
    nv = C.c_int64(); nf = C.c_int64()
    rc = _r.ref_mesh_clean(xyz.ctypes.data, rgb.ctypes.data if rgb is not None else None, nV, tri.ctypes.data, nF, merge_threshold,
                           (1 if merge else 0) | (2 if dedup else 0), ox.ctypes.data, oc.ctypes.data, ot.ctypes.data, C.addressof(nv), C.addressof(nf))
    if rc == -1:
        raise OracleRefusal("mLib threw")
    return ox[:nv.value].copy(), (oc[:nv.value].copy() if rgb is not None else None), ot[:nf.value].copy()
