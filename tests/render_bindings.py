"""ctypes bindings for the render oracle (oracle/_build/liboracle_render.so, DESIGN.md §6i).  TEST INFRASTRUCTURE: only
tests/, __graft_entry__.smoke() and scripts/bench_render.py import this."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle/_build/liboracle_render.so")
NO_HIT = 0xFFFFFFFF

_o = None


def _lib():
    global _o
    if _o is None:
        if not os.path.exists(ORACLE):
            raise FileNotFoundError(f"{ORACLE} missing — run `make oracle` (oracle/render.mk)")
        _o = C.CDLL(ORACLE)
        _o.oracle_render.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                     C.c_uint32, C.c_float, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                     C.c_void_p, C.c_void_p]
        _o.oracle_first_hits.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_float, C.c_int,
                                         C.c_void_p, C.c_void_p]
        _o.oracle_render_tables.argtypes = [C.c_void_p, C.c_void_p]
    return _o


def tables():
    """(lin float32[256], thr float32[255]): sRGB byte -> linear, and the tonemap thresholds."""
    lin = np.zeros(256, np.float32); thr = np.zeros(255, np.float32)
    _lib().oracle_render_tables(lin.ctypes.data, thr.ctypes.data)
    return lin, thr


def oracle_render(xyz, rgb, tri, params, cams, mode=1, rect=None):
    """The oracle's RGBA (n_views, h, w, 4) of the pixel rectangle rect = (x0, y0, w, h) (default: the film) and its
    counters {primary_rays, secondary_rays, primary_hits}.  cams: RenderCamera list; mode 0 brute force, 1 its own BVH."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3); tri = np.ascontiguousarray(tri, np.uint32).reshape(-1, 3)
    if rgb is not None:
        rgb = np.ascontiguousarray(rgb, np.uint8).reshape(-1, 3)
    cam = np.ascontiguousarray(np.stack([c.as_array() for c in cams]), np.float32)
    x0, y0, w, h = rect if rect is not None else (0, 0, params.width, params.height)
    out = np.zeros((len(cams), h, w, 4), np.uint8)
    cnt = np.zeros(3, np.uint64)
    rc = _lib().oracle_render(xyz.ctypes.data, rgb.ctypes.data if rgb is not None else None, len(xyz), tri.ctypes.data, len(tri),
                              params.width, params.height, params.samples, params.integrator, params.max_depth, params.exposure,
                              cam.ctypes.data, len(cams), x0, y0, w, h, mode, out.ctypes.data, cnt.ctypes.data)
    assert rc == 0, "oracle out of memory"
    return out, dict(zip(("primary_rays", "secondary_rays", "primary_hits"), (int(v) for v in cnt)))


def first_hits(xyz, tri, o, d, tmin=0.0, mode=1):
    """(face uint32[n] (NO_HIT for none), t float32[n]) of the rays o + t d, t > tmin."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3); tri = np.ascontiguousarray(tri, np.uint32).reshape(-1, 3)
    o = np.ascontiguousarray(o, np.float32).reshape(-1, 3); d = np.ascontiguousarray(d, np.float32).reshape(-1, 3)
    face = np.zeros(len(o), np.uint32); t = np.zeros(len(o), np.float32)
    rc = _lib().oracle_first_hits(xyz.ctypes.data, tri.ctypes.data, len(tri), o.ctypes.data, d.ctypes.data, len(o), tmin, mode,
                                  face.ctypes.data, t.ctypes.data)
    assert rc == 0
    return face, t
