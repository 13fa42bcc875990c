"""ctypes bindings for the decimation oracle (oracle/_build/liboracle_meshsimplify.so, DESIGN.md §6g).
TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and scripts/bench_meshclean.py import this."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import meshclean_bindings as mb

ROOT = mb.ROOT
ORACLE = os.path.join(ROOT, "oracle/_build/liboracle_meshsimplify.so")
# counters[] of oracle_mesh_simplify, in order (the integer fields of scn_mesh_simplify_report_t after the four sizes)
COUNTERS = ["target_faces", "rounds", "collapses", "faces_collapsed", "autoclean_duplicate_faces", "max_vertex_faces"]
BATCHED, ONE_AT_A_TIME = 0, 1

_o = None


class CommutationError(AssertionError):
    pass


def _lib():
    global _o
    if _o is None:
        _o = mb._lib(ORACLE)
        _o.oracle_mesh_simplify.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_uint64, C.c_double, C.c_double,
                                            C.c_int, C.c_int64] + [C.c_void_p] * 9
    return _o


def _call(xyz, tri, rgb, target_faces, target_perc, quality_thr, mode, max_rounds):
    xyz, tri, rgb = mb._prep(xyz, tri, rgb)
    nV, nF = len(xyz), len(tri)
    ox = np.zeros((max(nV, 1), 3), np.float32); oc = np.zeros((max(nV, 1), 3), np.uint8); ot = np.zeros((max(nF, 1), 3), np.uint32)
    fa = np.zeros(max(nF, 1), np.uint8); q = np.zeros((max(nV, 1), 10), np.float64); cost = np.zeros(max(nF, 1), np.float64)
    nv = C.c_int64(); nf = C.c_int64(); cnt = np.zeros(len(COUNTERS), np.uint64)
    rc = _lib().oracle_mesh_simplify(xyz.ctypes.data, rgb.ctypes.data if rgb is not None else None, nV, tri.ctypes.data, nF, target_faces,
                                     target_perc, quality_thr, mode, max_rounds, ox.ctypes.data, oc.ctypes.data, ot.ctypes.data,
                                     C.addressof(nv), C.addressof(nf), cnt.ctypes.data, fa.ctypes.data, q.ctypes.data, cost.ctypes.data)
    if rc == -1:
        raise mb.OracleRefusal("refused")
    if rc == -3:
        raise CommutationError("a round's collapses do not commute")
    assert rc == 0, rc
    counters = dict(zip(COUNTERS, map(int, cnt)))
    return ox, oc, ot, nv.value, nf.value, counters, fa, q, cost


def oracle_simplify(xyz, tri, rgb=None, target_faces=0, target_perc=0.2, quality_thr=0.3, after=None):
    """The whole filter with AutoClean, then (if `after`, a dict of oracle_clean keyword arguments) the clean filters:
    (xyz, rgb or None, tri, counters dict, clean counters dict or None)."""
    ox, oc, ot, nv, nf, cnt, _, _, _ = _call(xyz, tri, rgb, target_faces, target_perc, quality_thr, BATCHED, -1)
    x, c, t = ox[:nv].copy(), (oc[:nv].copy() if rgb is not None else None), ot[:nf].copy()
    if after is None:
        return x, c, t, cnt, None
    x, c, t, ccnt = mb.oracle_clean(x, t, c, **after)
    return x, c, t, cnt, ccnt


def oracle_rounds(xyz, tri, rounds, mode=BATCHED, target_faces=0, target_perc=0.2, quality_thr=0.3):
    """State after `rounds` rounds, before AutoClean: dict of positions (all vertices), faces (all, renamed), alive flags,
    quadrics, the costs of the applied collapses in order, and the counters."""
    ox, _, ot, nv, nf, cnt, fa, q, cost = _call(xyz, tri, None, target_faces, target_perc, quality_thr, mode, rounds)
    nF = len(np.asarray(tri).reshape(-1, 3))
    return {"xyz": ox[:nv].copy(), "tri": ot[:nF].copy(), "alive": fa[:nF].astype(bool), "quadrics": q[:nv].copy(),
            "costs": cost[:cnt["collapses"]].copy(), "counters": cnt}
