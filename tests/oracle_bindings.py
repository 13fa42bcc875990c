"""ctypes bindings for the CPU oracles (oracle/_build) and the compiled reference (oracle/_ref).
TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and bench.py's CPU legs import this."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGE_DTYPE = np.dtype([("w", "<f4"), ("a", "<i4"), ("b", "<i4")])
VOXEL_DTYPE = np.dtype([("sdf", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1"), ("w", "u1")])


def _load(rel):
    p = os.path.join(ROOT, rel)
    if not os.path.exists(p):
        raise FileNotFoundError(f"{p} missing — run `make oracle` (and `make -C oracle ref` where /root/reference exists)")
    return C.CDLL(p)


class OracleTsdfParams(C.Structure):
    _fields_ = [("voxel_size", C.c_float), ("trunc_base", C.c_float), ("trunc_scale", C.c_float),
                ("depth_min", C.c_float), ("depth_max", C.c_float), ("max_integration_distance", C.c_float),
                ("weight_sample", C.c_uint32), ("weight_max", C.c_uint32),
                ("width", C.c_uint32), ("height", C.c_uint32), ("depth_shift", C.c_float)]


_seg = _tsdf = _refseg = _refsens = None


def seg_oracle():
    global _seg
    if _seg is None:
        _seg = _load("oracle/_build/liboracle_seg.so")
        _seg.oracle_segment_arrays.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_float, C.c_int32] + [C.c_void_p] * 4
        _seg.oracle_seg_sort_edges.argtypes = [C.c_void_p, C.c_int64]
        _seg.oracle_seg_build_edges.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    return _seg


def oracle_segment(xyz, tri, kthr=0.01, seg_min=20, want_debug=False):
    xyz = np.ascontiguousarray(xyz, np.float32); tri = np.ascontiguousarray(tri, np.uint32)
    nV, nF = len(xyz), len(tri)
    out = np.zeros(nV, np.int32)
    pre = np.zeros(3 * nF, EDGE_DTYPE); srt = np.zeros(3 * nF, EDGE_DTYPE); roots = np.zeros(nV, np.int32)
    rc = seg_oracle().oracle_segment_arrays(xyz.ctypes.data, nV, tri.ctypes.data, nF, kthr, seg_min, out.ctypes.data,
                                            pre.ctypes.data, srt.ctypes.data, roots.ctypes.data)
    assert rc == 0
    if want_debug:
        nrm = np.zeros((nV, 3), np.float32); e2 = np.zeros(3 * nF, EDGE_DTYPE)
        seg_oracle().oracle_seg_build_edges(xyz.ctypes.data, nV, tri.ctypes.data, nF, e2.ctypes.data, nrm.ctypes.data)
        return out, pre, srt, roots, nrm
    return out


def ref_segmentator():
    global _refseg
    if _refseg is None:
        _refseg = _load("oracle/_ref/libref_segmentator.so")
        _refseg.ref_segment_file.restype = C.c_int64
        _refseg.ref_segment_file.argtypes = [C.c_char_p, C.c_float, C.c_int, C.c_void_p, C.c_int64]
        _refseg.ref_segment_graph.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
    return _refseg


def ref_segment_file(path, n_verts, kthr=0.01, seg_min=20):
    out = np.zeros(n_verts, np.int32)
    n = ref_segmentator().ref_segment_file(str(path).encode(), kthr, seg_min, out.ctypes.data, n_verts)
    assert n == n_verts, (n, n_verts)
    return out


def tsdf_oracle_lib():
    global _tsdf
    if _tsdf is None:
        _tsdf = _load("oracle/_build/liboracle_tsdf.so")
        _tsdf.oracle_tsdf_create.restype = C.c_void_p
        _tsdf.oracle_tsdf_create.argtypes = [C.c_void_p, C.c_int]
        _tsdf.oracle_tsdf_destroy.argtypes = [C.c_void_p]
        _tsdf.oracle_tsdf_integrate.argtypes = [C.c_void_p] * 5
        _tsdf.oracle_tsdf_num_blocks.restype = C.c_uint64
        _tsdf.oracle_tsdf_num_blocks.argtypes = [C.c_void_p]
        _tsdf.oracle_tsdf_counters.argtypes = [C.c_void_p, C.c_void_p]
        _tsdf.oracle_tsdf_export.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _tsdf.oracle_tsdf_import.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        _tsdf.oracle_tsdf_extract_mesh.argtypes = [C.c_void_p, C.c_float] + [C.c_void_p] * 5
        _tsdf.oracle_free.argtypes = [C.c_void_p]
        _tsdf.oracle_mc_table.argtypes = [C.c_void_p, C.c_void_p]
        _tsdf.oracle_tsdf_integrate_metres.argtypes = [C.c_void_p] * 5
        _tsdf.oracle_bilateral_filter.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p]
    return _tsdf


class OracleTsdf:
    """Scalar CPU statement of TSDF spec v1 (oracle/tsdf_oracle.c)."""

    def __init__(self, params, threads: int = 1):
        p = OracleTsdfParams()
        for f, _ in OracleTsdfParams._fields_:
            setattr(p, f, getattr(params, f))
        self._p = p
        self._h = tsdf_oracle_lib().oracle_tsdf_create(C.byref(p), threads)

    def integrate(self, depth, rgb, cam2world, K):
        depth = np.ascontiguousarray(depth, np.uint16)
        T = np.ascontiguousarray(cam2world, np.float32); Kc = np.ascontiguousarray(K, np.float32)
        rp = None
        if rgb is not None:
            rgb = np.ascontiguousarray(rgb, np.uint8); rp = rgb.ctypes.data
        return tsdf_oracle_lib().oracle_tsdf_integrate(self._h, depth.ctypes.data, rp, T.ctypes.data, Kc.ctypes.data)

    def integrate_metres(self, metres, rgb, cam2world, K):
        m = np.ascontiguousarray(metres, np.float32)
        T = np.ascontiguousarray(cam2world, np.float32); Kc = np.ascontiguousarray(K, np.float32)
        rp = None
        if rgb is not None:
            rgb = np.ascontiguousarray(rgb, np.uint8); rp = rgb.ctypes.data
        return tsdf_oracle_lib().oracle_tsdf_integrate_metres(self._h, m.ctypes.data, rp, T.ctypes.data, Kc.ctypes.data)

    def counters(self):
        c = np.zeros(6, np.uint64)
        tsdf_oracle_lib().oracle_tsdf_counters(self._h, c.ctypes.data)
        return dict(last_updated=int(c[0]), last_touched=int(c[1]), total_updated=int(c[2]),
                    total_touched=int(c[3]), frames_done=int(c[4]), frames_skipped=int(c[5]))

    def export(self):
        n = tsdf_oracle_lib().oracle_tsdf_num_blocks(self._h)
        xyz = np.zeros((n, 3), np.int32); vox = np.zeros((n, 512), VOXEL_DTYPE)
        if n:
            tsdf_oracle_lib().oracle_tsdf_export(self._h, xyz.ctypes.data, vox.ctypes.data)
        return xyz, vox

    def import_blocks(self, block_xyz, voxels):
        """The inverse of export: adds blocks (int32 [n,3], VOXEL_DTYPE [n,512]); raises ValueError, volume unchanged,
        for a coordinate outside the key range or a block given twice or already present."""
        xyz = np.ascontiguousarray(block_xyz, np.int32).reshape(-1, 3)
        vox = np.ascontiguousarray(voxels, VOXEL_DTYPE).reshape(-1, 512)
        assert len(xyz) == len(vox)
        if tsdf_oracle_lib().oracle_tsdf_import(self._h, xyz.ctypes.data, vox.ctypes.data, len(xyz)) != 0:
            raise ValueError("oracle_tsdf_import refused the blocks")

    def extract_mesh(self, thresh_factor: float = 10.0):
        L = tsdf_oracle_lib()
        xyz = C.POINTER(C.c_float)(); rgb = C.POINTER(C.c_uint8)(); tri = C.POINTER(C.c_uint32)()
        nv = C.c_uint64(); nf = C.c_uint64()
        L.oracle_tsdf_extract_mesh(self._h, thresh_factor, C.byref(xyz), C.byref(rgb), C.byref(tri), C.byref(nv), C.byref(nf))
        V, F = nv.value, nf.value
        a = np.ctypeslib.as_array(xyz, (max(V * 3, 1),))[: V * 3].copy().reshape(-1, 3)
        c = np.ctypeslib.as_array(rgb, (max(V * 3, 1),))[: V * 3].copy().reshape(-1, 3)
        t = np.ctypeslib.as_array(tri, (max(F * 3, 1),))[: F * 3].copy().reshape(-1, 3)
        for p in (xyz, rgb, tri):
            L.oracle_free(p)
        return a, c, t

    def close(self):
        if self._h:
            tsdf_oracle_lib().oracle_tsdf_destroy(self._h); self._h = None

    __del__ = close


def oracle_bilateral(depth, depth_shift, sigma_d, sigma_r):
    depth = np.ascontiguousarray(depth, np.uint16)
    out = np.zeros(depth.shape, np.float32)
    tsdf_oracle_lib().oracle_bilateral_filter(depth.ctypes.data, depth.shape[1], depth.shape[0], depth_shift, sigma_d, sigma_r, out.ctypes.data)
    return out


# ---- segs.json consumers (oracle/segs_oracle.c, oracle/ref_shim_mlib.cpp) -------------------------------------
_segs = _refmlib = None


def segs_oracle():
    global _segs
    if _segs is None:
        _segs = _load("oracle/_build/liboracle_segs.so")
        _segs.oracle_tri_area_mlib.restype = C.c_float
        _segs.oracle_tri_area_mlib.argtypes = [C.c_void_p] * 3
        _segs.oracle_segs_aggregate.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 5
        _segs.oracle_objects_per_vertex.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        _segs.oracle_vertex_normals_mlib.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        _segs.oracle_propagate_labels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p]
    return _segs


def ref_mlib():
    global _refmlib
    if _refmlib is None:
        _refmlib = _load("oracle/_ref/libref_mlib.so")
        _refmlib.ref_tri_area.restype = C.c_float
        _refmlib.ref_tri_area.argtypes = [C.c_void_p] * 3
        _refmlib.ref_vertex_normals.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    return _refmlib


def oracle_segs_aggregate(seg, xyz=None, tri=None):
    seg = np.ascontiguousarray(seg, np.uint32); nV = len(seg)
    want = xyz is not None
    if want:
        xyz = np.ascontiguousarray(xyz, np.float32); tri = np.ascontiguousarray(tri, np.uint32)
    ids = np.zeros(max(nV, 1), np.uint32); off = np.zeros(nV + 1, np.uint64); vid = np.zeros(max(nV, 1), np.uint32)
    area = np.zeros(max(nV, 1), np.float32); nS = C.c_int64()
    segs_oracle().oracle_segs_aggregate(seg.ctypes.data, nV, xyz.ctypes.data if want else None, tri.ctypes.data if want else None,
                                        len(tri) if want else 0, ids.ctypes.data, C.addressof(nS), off.ctypes.data, vid.ctypes.data,
                                        area.ctypes.data if want else None)
    n = nS.value
    return dict(seg_ids=ids[:n].copy(), offsets=off[:n + 1].copy(), vert_ids=vid[:nV].copy(), area=area[:n].copy() if want else None)


def oracle_objects_per_vertex(seg, groups):
    seg = np.ascontiguousarray(seg, np.uint32)
    flat = np.ascontiguousarray(np.concatenate([np.asarray(list(g), np.uint32) for g in groups]) if groups else np.zeros(1, np.uint32), np.uint32)
    offs = np.zeros(len(groups) + 1, np.uint64); offs[1:] = np.cumsum([len(list(g)) for g in groups]) if groups else []
    out = np.zeros(len(seg), np.uint32)
    segs_oracle().oracle_objects_per_vertex(seg.ctypes.data, len(seg), flat.ctypes.data, offs.ctypes.data, len(groups), out.ctypes.data)
    return out


def oracle_vertex_normals_mlib(xyz, tri):
    xyz = np.ascontiguousarray(xyz, np.float32); tri = np.ascontiguousarray(tri, np.uint32)
    out = np.zeros((len(xyz), 3), np.float32)
    segs_oracle().oracle_vertex_normals_mlib(xyz.ctypes.data, len(xyz), tri.ctypes.data, len(tri), out.ctypes.data)
    return out


def ref_vertex_normals_mlib(xyz, tri):
    xyz = np.ascontiguousarray(xyz, np.float32); tri = np.ascontiguousarray(tri, np.uint32)
    out = np.zeros((len(xyz), 3), np.float32)
    ref_mlib().ref_vertex_normals(xyz.ctypes.data, len(xyz), tri.ctypes.data, len(tri), out.ctypes.data)
    return out


def oracle_propagate_labels(sx, sn, so, dx, dn, thresh=0.5):
    sx = np.ascontiguousarray(sx, np.float32); sn = np.ascontiguousarray(sn, np.float32); so = np.ascontiguousarray(so, np.uint32)
    dx = np.ascontiguousarray(dx, np.float32); dn = np.ascontiguousarray(dn, np.float32)
    out = np.zeros(len(dx), np.uint32); edge = np.zeros(len(dx), np.uint8)
    segs_oracle().oracle_propagate_labels(sx.ctypes.data, sn.ctypes.data, so.ctypes.data, len(sx), dx.ctypes.data, dn.ctypes.data, len(dx),
                                          thresh, out.ctypes.data, edge.ctypes.data)
    return out, edge.astype(bool)
