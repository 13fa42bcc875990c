"""Decimation spec (DESIGN.md §6g) on the CPU: the oracle's quadric algebra against an independent numpy statement, the
commutation of a round's collapses (batched vs one collapse at a time), planar grids, target accounting, the simplify.mlx reader
and the report binding."""
import ctypes as C
import os

import numpy as np
import pytest

import meshclean_bindings as mb
import meshsimplify_bindings as sb
from meshsimplify_cases import fan, grid, soup, strip
from scannet_b200 import ScnError, meshsimplify

GOLDEN = os.path.join(mb.ROOT, "tests", "golden")


def plane_sq_dist_sum(xyz, tri, verts, p):
    """sum over the corners at `verts` of 2*area(f) * dist(p, plane(f))^2, in float64 from the float32 corners"""
    x = xyz.astype(np.float64)
    tot = 0.0
    for f in tri:
        p0, p1, p2 = x[f[0]], x[f[1]], x[f[2]]
        n = np.cross(p1 - p0, p2 - p0)
        ln = np.linalg.norm(n)
        if ln == 0:
            continue
        d = np.dot(n / ln, np.asarray(p, np.float64) - p0)
        tot += sum(ln * d * d for c in f if c in verts)
    return tot


def collapses_of_round(tri0, st):
    """(b -> a) of the first round, read off the surviving faces' renamed corners"""
    out = {}
    for f0, f, alive in zip(tri0, st["tri"], st["alive"]):
        if alive:
            for u, v in zip(f0, f):
                if u != v:
                    out[int(u)] = int(v)
    return out


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_error_is_the_area_weighted_plane_distance(built, seed):
    xyz, tri = grid(24, 20, seed=seed, spacing=1.0, z_noise=0.2)
    st = sb.oracle_rounds(xyz, tri, 1, quality_thr=0.0)                 # no penalty: cost = max(err, 1e-15)
    pairs = collapses_of_round(tri, st)
    costs = st["costs"]
    checked = 0
    for b, a in pairs.items():
        want = plane_sq_dist_sum(xyz, tri, {a, b}, st["xyz"][a])
        if want < 1e-6:                                                 # cancellation dominates near-zero errors
            continue
        checked += 1
        # 1e-9 relative, plus the cancellation of p*'Qp* at coordinates ~10 (terms ~1e2, binary64)
        assert np.min(np.abs(costs - want)) <= 1e-9 * want + 1e-12, (a, b, want, costs)
    assert checked >= 3


def quad_err(q, p):
    x, y, z = (float(v) for v in p)
    return (q[0] * x * x + 2 * q[1] * x * y + 2 * q[2] * x * z + 2 * q[3] * x + q[4] * y * y + 2 * q[5] * y * z + 2 * q[6] * y
            + q[7] * z * z + 2 * q[8] * z + q[9])


@pytest.mark.parametrize("seed", [3, 4])
def test_accepted_optimum_is_no_worse_than_endpoints_and_midpoint(built, seed):
    xyz, tri = grid(10, 10, seed=seed, spacing=1.0, z_noise=0.2)
    q0 = sb.oracle_rounds(xyz, tri, 0)["quadrics"]
    st = sb.oracle_rounds(xyz, tri, 1, quality_thr=0.0)
    n_opt = 0
    for b, a in collapses_of_round(tri, st).items():
        q = q0[a] + q0[b]
        p = st["xyz"][a]
        pa, pb = xyz[a], xyz[b]
        mid = (0.5 * (pa.astype(np.float64) + pb)).astype(np.float32)
        if any((p == c).all() for c in (pa, pb, mid)):
            continue
        n_opt += 1
        others = min(quad_err(q, c) for c in (pa, pb, mid))
        delta = 2.0 ** -24 * float(np.abs(p).max()) * np.sqrt(3)          # rounding of p* to binary32
        slack = (q[0] + q[4] + q[7]) * delta * delta + 1e-12 * abs(others)
        assert quad_err(q, p) <= others + slack
    assert n_opt >= 3


CASES = {
    "grid": lambda: grid(12, 11, seed=5),
    "fan": lambda: fan(40, seed=1),
    "strip": lambda: strip(60, seed=2),
    "soup": lambda: soup(30, 90, seed=3),
    "grid_flat": lambda: grid(9, 9, seed=6, z0=0.25),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("thr", [0.0, 0.3, 1.0])
def test_round_equals_one_collapse_at_a_time(built, case, thr):
    xyz, tri = CASES[case]()
    final = sb.oracle_rounds(xyz, tri, 10 ** 6, target_perc=0.0, target_faces=0, quality_thr=thr)["counters"]["rounds"]
    assert final >= 1
    for r in range(1, min(final, 12) + 1):
        a = sb.oracle_rounds(xyz, tri, r, sb.BATCHED, target_perc=0.0, target_faces=0, quality_thr=thr)
        b = sb.oracle_rounds(xyz, tri, r, sb.ONE_AT_A_TIME, target_perc=0.0, target_faces=0, quality_thr=thr)
        assert a["xyz"].tobytes() == b["xyz"].tobytes(), r
        assert a["quadrics"].tobytes() == b["quadrics"].tobytes(), r
        assert (a["alive"] == b["alive"]).all() and a["tri"][a["alive"]].tobytes() == b["tri"][b["alive"]].tobytes(), r
        assert a["costs"].tobytes() == b["costs"].tobytes(), r
        assert a["counters"] == b["counters"], r


def test_planar_grid_stays_on_its_plane(built):
    xyz, tri = grid(30, 25, seed=7, z0=0.25)
    ox, _, ot, cnt, _ = sb.oracle_simplify(xyz, tri)
    assert cnt["collapses"] > 0 and len(ot) <= cnt["target_faces"]
    assert (ox[:, 2] == np.float32(0.25)).all()


@pytest.mark.parametrize("perc", [0.5, 0.2, 0.05])
def test_target_is_met_and_the_last_collapse_was_needed(built, perc):
    xyz, tri = grid(20, 18, seed=8)                       # manifold: a collapse removes 1 or 2 faces
    _, _, ot, cnt, _ = sb.oracle_simplify(xyz, tri, target_perc=perc)
    target = int(np.floor(len(tri) * perc))
    assert cnt["target_faces"] == target
    left = len(tri) - cnt["faces_collapsed"]
    assert target - 1 <= left <= target                   # before the last collapse there were left + (1 or 2) > target faces
    assert len(ot) == left - cnt["autoclean_duplicate_faces"]


def test_target_at_or_above_the_face_count_only_compacts(built):
    xyz, tri = grid(6, 5, seed=9)
    extra = np.vstack([xyz, np.float32([[5, 5, 5], [6, 6, 6]])])          # two unreferenced vertices
    for kw in ({"target_perc": 1.0}, {"target_perc": 0.0, "target_faces": len(tri)}, {"target_perc": 0.0, "target_faces": 10 ** 9}):
        ox, _, ot, cnt, _ = sb.oracle_simplify(extra, tri, **kw)
        assert cnt["rounds"] == 0 and cnt["collapses"] == 0
        assert ox.tobytes() == xyz.tobytes() and ot.tobytes() == tri.tobytes()


def test_target_zero_collapses_until_nothing_is_left(built):
    xyz, tri = grid(7, 6, seed=10)
    ox, _, ot, cnt, _ = sb.oracle_simplify(xyz, tri, target_perc=0.0, target_faces=0)
    assert len(ot) == 0 and len(ox) == 0 and cnt["faces_collapsed"] == len(tri)


def test_oracle_refusals(built):
    xyz, tri = grid(4, 4)
    for kw in ({"target_perc": float("nan")}, {"target_perc": -0.1}, {"target_perc": 1.5}, {"quality_thr": -1.0}, {"quality_thr": float("nan")}):
        with pytest.raises(mb.OracleRefusal):
            sb.oracle_simplify(xyz, tri, **kw)
    bad = xyz.copy(); bad[3, 1] = np.inf
    with pytest.raises(mb.OracleRefusal):
        sb.oracle_simplify(bad, tri)
    with pytest.raises(mb.OracleRefusal):
        sb.oracle_simplify(xyz, np.array([[0, 1, len(xyz)]], np.uint32))


# ---- the script reader --------------------------------------------------------------------------------------------------
def test_params_from_simplify_mlx(built):
    p, a = meshsimplify.params_from_mlx(os.path.join(GOLDEN, "simplify.mlx"))
    assert (p.target_faces, p.target_perc, p.quality_thr) == (0, 0.2, 0.3)
    assert a.merge_threshold == np.float32(0.0010689) and a.min_piece_faces == 1000 and a.flags == 0
    d, da = meshsimplify.default_params()
    assert (d.target_faces, d.target_perc, d.quality_thr) == (0, 0.2, 0.3)
    assert (da.merge_threshold, da.min_piece_faces, da.min_piece_vertices, da.flags) == (a.merge_threshold, 1000, 0, 0)


FLIPS = [("PreserveBoundary", "false", "true"), ("PreserveNormal", "false", "true"), ("PreserveTopology", "false", "true"),
         ("OptimalPlacement", "true", "false"), ("PlanarQuadric", "false", "true"), ("QualityWeight", "false", "true"),
         ("AutoClean", "true", "false"), ("Selected", "false", "true"), ("BoundaryWeight", "1", "2")]


@pytest.mark.parametrize("name,old,new", FLIPS)
def test_unsupported_option_is_refused_by_name(built, tmp_path, name, old, new):
    src = open(os.path.join(GOLDEN, "simplify.mlx")).read()
    key = f'value="{old}"'
    i = src.index(f'name="{name}"')
    line_start = src.rindex("<Param", 0, i)
    line = src[line_start:src.index("/>", i)]
    assert key in line
    path = tmp_path / "s.mlx"
    path.write_text(src[:line_start] + line.replace(key, f'value="{new}"') + src[line_start + len(line):])
    with pytest.raises(ScnError) as e:
        meshsimplify.params_from_mlx(str(path))
    assert e.value.code == -6 and name in str(e.value)


def test_other_scripts_are_refused(built, tmp_path):
    for f in ("clean.mlx", "cleanLoRes.mlx"):
        with pytest.raises(ScnError) as e:
            meshsimplify.params_from_mlx(os.path.join(GOLDEN, f))
        assert e.value.code == -6
    src = open(os.path.join(GOLDEN, "simplify.mlx")).read()
    q = src[src.index(" <filter"):src.index("</filter>") + len("</filter>")]
    twice = tmp_path / "twice.mlx"
    twice.write_text(src.replace(q, q + "\n" + q))
    with pytest.raises(ScnError) as e:
        meshsimplify.params_from_mlx(str(twice))
    assert e.value.code == -6 and "Quadric Edge Collapse Decimation" in str(e.value)
    alone = tmp_path / "alone.mlx"
    alone.write_text("<!DOCTYPE FilterScript>\n<FilterScript>\n" + q + "\n</FilterScript>\n")
    p, a = meshsimplify.params_from_mlx(str(alone))
    assert p.target_perc == 0.2 and a.flags == mb.SKIP_MERGE | mb.SKIP_DEDUP | mb.SKIP_PIECES
    with pytest.raises(ScnError):
        meshsimplify.params_from_mlx(str(tmp_path / "missing.mlx"))


def test_report_binding_matches_the_library_struct(built):
    assert meshsimplify.report_sizeof() == C.sizeof(meshsimplify.SimplifyReport)
    assert meshsimplify.COUNTERS == sb.COUNTERS
