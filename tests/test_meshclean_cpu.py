"""CPU: the mesh-cleaning oracle (oracle/meshclean_oracle.c) pinned against the unmodified mLib MeshData operators
(oracle/_ref/libref_meshdata.so: mergeCloseVertices(t, false) and removeDuplicateFaces, compiled where they lie), hand-built
cases for the piece step (mLib's removeIsolatedVertices does not compile under g++, so that step is pinned to DESIGN §6f),
the MeshLab FilterScript reader and the colour-aware PLY loader (host code, no GPU needed)."""
import os

import numpy as np
import pytest

import meshclean_bindings as mb
from scannet_b200 import ScnError, meshclean

GOLDEN = os.path.join(mb.ROOT, "tests", "golden")


@pytest.fixture
def mlib_ref(built):
    """decided after build(), which compiles the shim where the reference tree exists"""
    if not mb.have_ref():
        pytest.skip("compiled mLib MeshData shim not present (built where the reference tree exists)")


needs_ref = pytest.mark.usefixtures("mlib_ref")


def pin(xyz, tri, rgb, t, steps):
    """oracle vs mLib, byte for byte, for one or both of the pinned steps"""
    flags = mb.SKIP_PIECES | (0 if "merge" in steps else mb.SKIP_MERGE) | (0 if "dedup" in steps else mb.SKIP_DEDUP)
    ox, oc, ot, cnt = mb.oracle_clean(xyz, tri, rgb, merge_threshold=t, flags=flags)
    rx, rc, rt = mb.ref_clean(xyz, tri, rgb, merge_threshold=t, merge="merge" in steps, dedup="dedup" in steps)
    assert ox.tobytes() == rx.tobytes()
    assert (oc is None and rc is None) or oc.tobytes() == rc.tobytes()
    assert ot.tobytes() == rt.tobytes()
    return ox, oc, ot, cnt


def random_faces(rng, nV, nF):
    tri = rng.integers(0, nV, (nF, 3)).astype(np.uint32)
    tri[::17, 1] = tri[::17, 0]                                            # degenerate
    tri[5::23] = tri[4::23][: len(tri[5::23])]                             # duplicates
    tri[7::29] = tri[6::29][: len(tri[7::29]), ::-1]                       # flipped duplicates
    return tri


@needs_ref
@pytest.mark.parametrize("t", [0.0005, 0.002, 0.01, 0.05])
def test_random_cloud_matches_mlib(built, t):
    rng = np.random.default_rng(int(t * 1e5))
    xyz = rng.uniform(-0.1, 0.1, (4000, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (4000, 3)).astype(np.uint8)
    tri = random_faces(rng, 4000, 6000)
    _, _, _, cnt = pin(xyz, tri, rgb, t, ("merge", "dedup"))
    pin(xyz, tri, rgb, t, ("merge",))
    pin(xyz, tri, rgb, t, ("dedup",))
    if t >= 0.01:
        assert cnt["vertices_merged"] > 0 and cnt["degenerate_faces"] > 0


@needs_ref
@pytest.mark.parametrize("jitter", [0.0, 0.2, 0.45])
def test_jittered_grid_matches_mlib(built, jitter):
    rng = np.random.default_rng(7)
    s = 0.004
    g = np.stack(np.meshgrid(*[np.arange(-12, 12)] * 3, indexing="ij"), -1).reshape(-1, 3) * s
    xyz = (g + rng.uniform(-jitter, jitter, g.shape) * s).astype(np.float32)
    xyz = xyz[rng.permutation(len(xyz))]
    tri = random_faces(rng, len(xyz), 20000)
    for t in (s * 0.5, s, s * 1.5):
        pin(xyz, tri, None, np.float32(t), ("merge", "dedup"))


@needs_ref
def test_cell_boundaries_and_signs_match_mlib(built):
    """coordinates at (k + 1/2) * t +- 1 ulp, the rounding point of toVirtualVoxelPos, with zero, -0 and negative values"""
    t = np.float32(0.01)
    base = (np.arange(-6, 6, dtype=np.float32) + np.float32(0.5)) * t
    vals = np.concatenate([base, np.nextafter(base, np.float32(np.inf)), np.nextafter(base, np.float32(-np.inf)),
                           np.array([0.0, -0.0, 1e-30, -1e-30], np.float32)]).astype(np.float32)
    rng = np.random.default_rng(3)
    xyz = rng.choice(vals, (3000, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (3000, 3)).astype(np.uint8)
    tri = random_faces(rng, 3000, 3000)
    for tt in (t, np.float32(0.0099), np.float32(0.0101)):
        pin(xyz, tri, rgb, tt, ("merge", "dedup"))


@needs_ref
def test_exact_threshold_does_not_merge(built):
    """d^2 == t*t exactly: the comparison is strict (meshData.cpp:186)"""
    t = np.float32(0.5)
    xyz = np.array([[0, 0, 0], [0.5, 0, 0], [0, -0.5, 0], [0.25, 0.25, 0.25], [-0.3, 0.4, 0]], np.float32)   # |v4| = 0.5
    tri = np.array([[0, 1, 2], [1, 2, 4]], np.uint32)
    ox, _, ot, cnt = pin(xyz, tri, None, t, ("merge", "dedup"))
    # vertex 3 is within 0.5 of vertex 0 (d^2 = 0.1875): it is the only one that merges
    assert len(ox) == 4 and cnt["vertices_merged"] == 1


@needs_ref
def test_faces_degenerate_duplicate_flipped(built):
    xyz = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0, 0, 1]], np.float32)
    tri = np.array([[0, 1, 2], [2, 1, 0], [1, 2, 0], [0, 0, 3], [1, 3, 2], [3, 3, 3], [0, 1, 2], [2, 3, 1], [4, 0, 1]], np.uint32)
    ox, _, ot, cnt = pin(xyz, tri, None, np.float32(0.1), ("merge", "dedup"))
    assert ot.tolist() == [[0, 1, 2], [1, 3, 2], [4, 0, 1]]
    assert cnt["degenerate_faces"] == 2 and cnt["duplicate_faces"] == 4
    # dedup alone keeps the degenerate faces (only the merge step removes them)
    _, _, ot2, _ = pin(xyz, tri, None, np.float32(0.1), ("dedup",))
    assert [0, 0, 3] in ot2.tolist() and [3, 3, 3] in ot2.tolist()


@needs_ref
@pytest.mark.parametrize("order", ["near_later", "near_first"])
def test_first_in_scan_order_is_not_the_nearest(built, order):
    """t = 1: v_a (cell x=0) and v_b (cell x=2) are representatives; v_c (cell x=1) is 0.95 from v_a, 0.75 from v_b.  The x = -1
    offset is scanned first, so v_c maps to v_a, which is neither the nearest nor (in near_first) the lowest-index one."""
    a, b, c = [0.2, 0, 0], [1.9, 0, 0], [1.15, 0, 0]
    xyz = np.array([a, b, c] if order == "near_later" else [b, a, c], np.float32)
    tri = np.array([[0, 1, 2]], np.uint32)
    ox, _, ot, _ = pin(xyz, tri, None, np.float32(1.0), ("merge",))
    assert len(ox) == 2
    ia = 0 if order == "near_later" else 1
    assert ot.shape == (0, 3)                                             # the only face became degenerate (c -> a)
    x2, _, t2, _ = mb.oracle_clean(np.vstack([xyz, [[5, 5, 5], [6, 5, 5]]]).astype(np.float32), np.array([[2, 3, 4]], np.uint32), None,
                                   merge_threshold=1.0, flags=mb.SKIP_PIECES | mb.SKIP_DEDUP)
    assert x2[t2[0, 0]].tolist() == xyz[ia].tolist()


def test_merge_refusals(built):
    xyz = np.zeros((3, 3), np.float32); tri = np.array([[0, 1, 2]], np.uint32)
    for t in (0.0, -1.0, float("nan")):
        with pytest.raises(mb.OracleRefusal):
            mb.oracle_clean(xyz, tri, merge_threshold=t)
    for bad in (np.inf, np.nan, 3e6):
        x = xyz.copy(); x[1, 2] = bad
        with pytest.raises(mb.OracleRefusal):
            mb.oracle_clean(x, tri, merge_threshold=0.001)                 # 3e6 / 0.001 >= 2^31
    with pytest.raises(mb.OracleRefusal):
        mb.oracle_clean(xyz, np.array([[0, 1, 3]], np.uint32), merge_threshold=0.001)
    # with the merge skipped the threshold and the coordinates are not looked at
    mb.oracle_clean(np.full((3, 3), np.inf, np.float32), tri, merge_threshold=0.0, flags=mb.SKIP_MERGE)


# ---- piece step: hand-built (DESIGN §6f) -------------------------------------------------------------------------------
def pieces(xyz, tri, min_v=0, min_f=0):
    return mb.oracle_clean(xyz, tri, None, min_piece_vertices=min_v, min_piece_faces=min_f, flags=mb.SKIP_MERGE | mb.SKIP_DEDUP)


def test_pieces_touching_at_a_vertex_are_one_piece(built):
    xyz = np.arange(24, dtype=np.float32).reshape(8, 3)
    tri = np.array([[0, 1, 2], [2, 3, 4], [5, 6, 7]], np.uint32)          # bow-tie through vertex 2, plus a lone triangle
    _, _, t, c = pieces(xyz, tri, min_v=5)
    assert t.tolist() == [[0, 1, 2], [2, 3, 4]] and c["pieces_total"] == 2 and c["pieces_removed"] == 1 and c["faces_in_removed_pieces"] == 1
    _, _, t, c = pieces(xyz, tri, min_v=6)
    assert len(t) == 0 and c["pieces_removed"] == 2
    _, _, t, c = pieces(xyz, tri, min_f=2)
    assert len(t) == 2
    _, _, t, c = pieces(xyz, tri, min_f=3)
    assert len(t) == 0
    _, _, t, c = pieces(xyz, tri, min_v=3, min_f=1)                       # both thresholds exactly at the lone triangle's size
    assert len(t) == 3
    _, _, t, c = pieces(xyz, tri, min_v=4, min_f=1)
    assert len(t) == 2


def test_pieces_vertex_count_includes_vertices_of_every_face(built):
    """a piece's size counts vertices, not faces: a fan of 4 faces has 6 vertices"""
    xyz = np.zeros((6, 3), np.float32)
    tri = np.array([[0, 1, 2], [0, 2, 3], [0, 3, 4], [0, 4, 5]], np.uint32)
    assert len(pieces(xyz, tri, min_v=6)[2]) == 4 and len(pieces(xyz, tri, min_v=7)[2]) == 0
    assert len(pieces(xyz, tri, min_f=4)[2]) == 4 and len(pieces(xyz, tri, min_f=5)[2]) == 0


def test_unreferenced_vertices_and_first_appearance_order(built):
    xyz = np.arange(21, dtype=np.float32).reshape(7, 3)
    rgb = np.arange(21, dtype=np.uint8).reshape(7, 3)
    tri = np.array([[5, 3, 4], [3, 1, 2], [5, 5, 1]], np.uint32)        # 0 and 6 unreferenced; a degenerate face passes through
    x, c, t, cnt = mb.oracle_clean(xyz, tri, rgb, min_piece_faces=0, flags=mb.SKIP_MERGE | mb.SKIP_DEDUP)
    assert t.tolist() == [[0, 1, 2], [1, 3, 4], [0, 0, 3]]
    assert x.tolist() == xyz[[5, 3, 4, 1, 2]].tolist() and c.tolist() == rgb[[5, 3, 4, 1, 2]].tolist()
    assert cnt["pieces_total"] == 1 and cnt["pieces_removed"] == 0


def test_everything_removed_and_empty(built):
    xyz = np.zeros((3, 3), np.float32)
    x, _, t, c = mb.oracle_clean(xyz, np.array([[0, 1, 2]], np.uint32), min_piece_faces=2, flags=mb.SKIP_MERGE)
    assert len(x) == 0 and len(t) == 0 and c["pieces_removed"] == 1
    x, _, t, c = mb.oracle_clean(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint32))
    assert len(x) == 0 and len(t) == 0
    x, _, t, c = mb.oracle_clean(np.ones((4, 3), np.float32), np.zeros((0, 3), np.uint32), flags=mb.SKIP_PIECES)
    assert len(x) == 1 and c["vertices_merged"] == 3 and c["largest_merge_component"] == 4 and c["merge_components"] == 1


# ---- FilterScript reader -------------------------------------------------------------------------------------------------
def test_params_from_clean_mlx(built):
    p = meshclean.params_from_mlx(os.path.join(GOLDEN, "clean.mlx"))
    assert p.merge_threshold == np.float32(0.0010689) and p.min_piece_faces == 7500 and p.min_piece_vertices == 0 and p.flags == 0
    d = meshclean.default_params()
    assert (d.merge_threshold, d.min_piece_faces, d.min_piece_vertices, d.flags) == (p.merge_threshold, 7500, 0, 0)


def test_params_from_clean_lores_mlx(built):
    p = meshclean.params_from_mlx(os.path.join(GOLDEN, "cleanLoRes.mlx"))
    assert p.merge_threshold == np.float32(0.0010689) and p.min_piece_faces == 1000 and p.flags == 0


def test_simplify_mlx_is_refused(built):
    with pytest.raises(ScnError, match="Quadric Edge Collapse Decimation") as e:
        meshclean.params_from_mlx(os.path.join(GOLDEN, "simplify.mlx"))
    assert e.value.code == -6


def test_partial_and_malformed_scripts(built, tmp_path):
    p = tmp_path / "dedup.mlx"
    p.write_text('<!DOCTYPE FilterScript>\n<FilterScript>\n <filter name="Remove Duplicate Faces"/>\n</FilterScript>\n')
    q = meshclean.params_from_mlx(str(p))
    assert q.flags == meshclean.SKIP_MERGE | meshclean.SKIP_PIECES
    p.write_text('<FilterScript><filter name="Remove Unreferenced Vertex"/><filter name="Merge Close Vertices">'
                 '<Param name="Threshold" value="0.002" type="RichAbsPerc"/></filter></FilterScript>')
    with pytest.raises(ScnError, match="order"):
        meshclean.params_from_mlx(str(p))
    p.write_text('<FilterScript><filter name="Merge Close Vertices"><Param name="Threshold" value="abc"/></filter></FilterScript>')
    with pytest.raises(ScnError, match="not a number"):
        meshclean.params_from_mlx(str(p))
    with pytest.raises(ScnError):
        meshclean.params_from_mlx(str(tmp_path / "missing.mlx"))


# ---- loader ---------------------------------------------------------------------------------------------------------------
def test_load_rgb_gates381(built):
    path = os.path.join(GOLDEN, "gates381.ply")
    x, c, t = meshclean.load_rgb(path)
    data = open(path, "rb").read()
    body = data[data.index(b"end_header\n") + len(b"end_header\n"):]
    v = np.frombuffer(body[: 5860 * 28], dtype=[("p", "<f4", (3,)), ("n", "<f4", (3,)), ("c", "u1", (4,))])
    f = np.frombuffer(body[5860 * 28:], dtype=[("k", "u1"), ("i", "<u4", (3,))])
    assert x.tobytes() == np.ascontiguousarray(v["p"]).tobytes() and c.tobytes() == np.ascontiguousarray(v["c"][:, :3]).tobytes()
    assert t.tobytes() == np.ascontiguousarray(f["i"]).tobytes() and len(t) == 10197
    assert len(np.unique(c.reshape(-1, 3), axis=0)) > 10


def test_load_rgb_without_colour_and_ascii(built, tmp_path):
    p = tmp_path / "plain.ply"
    p.write_text("ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\n"
                 "element face 1\nproperty list uchar int vertex_indices\nend_header\n0 0 0\n1 0 0\n0 1 0\n3 0 1 2\n")
    x, c, t = meshclean.load_rgb(str(p))
    assert c is None and x.tolist() == [[0, 0, 0], [1, 0, 0], [0, 1, 0]] and t.tolist() == [[0, 1, 2]]
    q = tmp_path / "col.ply"
    q.write_text("ply\nformat ascii 1.0\nelement vertex 2\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\n"
                 "property uchar green\nproperty uchar blue\nelement face 0\nproperty list uchar int vertex_indices\nend_header\n"
                 "0 0 0 1 2 3\n1 0 0 250 251 252\n")
    x, c, t = meshclean.load_rgb(str(q))
    assert c.tolist() == [[1, 2, 3], [250, 251, 252]] and len(t) == 0


def test_report_binding_matches_the_library_struct(built):
    import ctypes as C
    assert meshclean.report_sizeof() == C.sizeof(meshclean.CleanReport)
    assert meshclean.COUNTERS == mb.COUNTERS
