"""The float64 statement of the marching-cubes spec (tests/mc_reference.py) against the CPU oracle (oracle/tsdf_oracle.c), on
designed volumes imported into the oracle block by block.  The GPU tests (test_mc_designed_gpu.py) hold the CUDA mesh to
both; this file pins the statement itself without a GPU."""
import numpy as np
import pytest

import mc_reference as mr
import mc_volumes as mv
import oracle_bindings as ob
from scannet_b200 import tsdf


def params():
    return tsdf.default_params(width=64, height=48, max_blocks=1 << 15, hash_slots=1 << 16)


def oracle_mesh(xyz, vox):
    o = ob.OracleTsdf(params())
    o.import_blocks(xyz, vox)
    m = o.extract_mesh()
    o.close()
    return m


def test_reference_triangulation_equals_oracle_table(built):
    n = np.zeros(256, np.uint8); t = np.zeros((256, 36), np.uint8)
    ob.tsdf_oracle_lib().oracle_mc_table(n.ctypes.data, t.ctypes.data)
    NT, TT = mr.table()
    bad = [cs for cs in range(256) if NT[cs] != n[cs] or (TT[cs].ravel() != t[cs]).any()]
    assert not bad, f"cases whose triangulation differs from the spec: {bad}"
    assert NT[0] == NT[255] == 0 and (NT[1:255] > 0).all()


@pytest.mark.parametrize("name", ["atlas", "boundary_values", "seams_and_keys", "no_crossing", "all_unusable", "sphere"])
def test_reference_equals_oracle(built, name):
    xyz, vox = getattr(mv, name)()
    ref = mr.extract(xyz, vox, mv.THR, mv.VS)
    mr.check(ref, *oracle_mesh(xyz, vox), mv.VS)


def test_atlas_has_every_case_at_every_position(built):
    xyz, vox = mv.atlas()
    ref = mr.extract(xyz, vox, mv.THR, mv.VS)
    assert len(ref["valid_case"]) == 2048                                 # the designed cubes and no other
    kind = ((ref["valid_g"] & 7) == 7).astype(int) @ np.array([1, 2, 4])
    for p in range(8):
        assert sorted(ref["valid_case"][kind == p].tolist()) == list(range(256)), mv.POSITION_NAMES[p]
    emitted = {tuple(g) for g in ref["cube"].tolist()}
    assert len(emitted) == 2048 - 16                                      # every cube but cases 0 and 255 emits


def test_boundary_values_spec(built):
    xyz, vox = mv.boundary_values()
    ref = mr.extract(xyz, vox, mv.THR, mv.VS)
    g = (8 * xyz[:, None, :].astype(np.int64) + np.stack([np.arange(512) & 7, (np.arange(512) >> 3) & 7, np.arange(512) >> 6], 1))
    s = vox["sdf"]; w = vox["w"]
    unusable = (w == 0) | (np.abs(s) > mv.THR)
    assert ((np.abs(s) == mv.THR_UP) & (w > 0)).any() and ((s < 0) & (w == 0)).any()
    bad = {tuple(v) for v in g[unusable].tolist()}
    ends = [tuple(e[:3]) for e in ref["edge"].tolist()] + [tuple(e[:3] + np.eye(3, dtype=int)[e[3]]) for e in ref["edge"]]
    assert not bad.intersection(ends), "a vertex on an edge that ends at an unusable voxel"
    # +0 and -0 are outside: a cube whose corners are all +-0 but one is case 1 << that corner
    zero_cubes = [c for c, k in zip(ref["valid_g"].tolist(), ref["valid_case"].tolist()) if k in (1 << 3, 1 << 5 | 1 << 6)]
    assert len(zero_cubes) >= 1
    assert (ref["rgb_lo"] != ref["rgb_hi"]).any(), "no colour tie was produced"


def test_oracle_import_refuses_and_leaves_the_volume(built):
    xyz, vox = mv.boundary_values()
    o = ob.OracleTsdf(params())
    o.import_blocks(xyz[:10], vox[:10])
    before = o.export()
    for bx, bv in [(np.array([[1 << 20, 0, 0]]), vox[:1]), (np.array([[0, -(1 << 20) - 1, 0]]), vox[:1]),
                   (np.concatenate([xyz[10:12], xyz[11:12]]), vox[10:13]), (xyz[9:11], vox[9:11])]:
        with pytest.raises(ValueError):
            o.import_blocks(bx, bv)
        after = o.export()
        assert after[0].tobytes() == before[0].tobytes() and after[1].tobytes() == before[1].tobytes()
    o.import_blocks(xyz[10:], vox[10:])
    ex, ev = o.export()
    order = np.argsort(mr.pack(xyz))
    assert ex.tobytes() == xyz[order].tobytes() and ev.tobytes() == vox[order].tobytes()
