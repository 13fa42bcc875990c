"""Marching cubes on the GPU (scn_tsdf_extract_mesh) on volumes built voxel by voxel and put on the device with
scn_tsdf_upload_blocks: every cube case at every block-seam position, boundary values, key-range edges, closed analytic
surfaces, degenerate volumes and one volume large enough for three-level scans.  Each mesh is held to
  - the CPU oracle, bit for bit (the same volume imported into oracle/tsdf_oracle.c),
  - the float64 statement of the spec (tests/mc_reference.py): the same triangles as lattice edges in the same order,
    vertices within 2 ulp of the float64 crossing, colours inside their rounding interval,
  - itself, with the blocks uploaded in another order.
The round-trip tests check upload as a volume restore: download, upload into a fresh volume, integrate on."""
import numpy as np
import pytest

import mc_reference as mr
import mc_volumes as mv
import oracle_bindings as ob
from scannet_b200 import ScnError, synth, tsdf

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAPACITY = -1, -5


def params(**kw):
    base = dict(width=64, height=48, max_blocks=1 << 15, hash_slots=1 << 16)
    base.update(kw)
    return tsdf.default_params(**base)


def gpu_mesh(xyz, vox, p=None):
    vol = tsdf.TsdfVolume(p or params(), device=0)
    vol.upload_blocks(xyz, vox)
    m = vol.extract_mesh()
    vol.close()
    return m


def same_bytes(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b)) and all(x.shape == y.shape for x, y in zip(a, b))


def three_way(xyz, vox, p=None):
    """GPU mesh == oracle mesh bit for bit; GPU mesh matches the float64 spec; a shuffled upload gives the same bytes"""
    g = gpu_mesh(xyz, vox, p)
    o = ob.OracleTsdf(p or params())
    o.import_blocks(xyz, vox)
    om = o.extract_mesh()
    o.close()
    assert g[0].view(np.uint32).tobytes() == om[0].view(np.uint32).tobytes(), "vertex positions differ from the oracle"
    assert g[1].tobytes() == om[1].tobytes(), "vertex colours differ from the oracle"
    assert g[2].shape == om[2].shape and g[2].tobytes() == om[2].tobytes(), "triangles differ from the oracle"
    ref = mr.extract(xyz, vox, mv.THR, mv.VS)
    mr.check(ref, *g, mv.VS)
    # every valid cube with a sign change emitted triangles
    nonempty = (ref["valid_case"] != 0) & (ref["valid_case"] != 255)
    assert len(np.unique(ref["cube"], axis=0)) == int(nonempty.sum())
    perm = np.random.default_rng(len(xyz)).permutation(len(xyz))
    assert same_bytes(gpu_mesh(xyz[perm], vox[perm], p), g), "the mesh depends on the upload order"
    return g, ref


def test_case_atlas(built):
    xyz, vox = mv.atlas()
    _, ref = three_way(xyz, vox)
    assert len(ref["valid_case"]) == 2048
    emitted = {tuple(c) for c in ref["cube"].tolist()}
    kind = ((ref["valid_g"] & 7) == 7).astype(int) @ np.array([1, 2, 4])
    for p in range(8):
        at = [(tuple(g), k) for g, k, q in zip(ref["valid_g"].tolist(), ref["valid_case"].tolist(), kind) if q == p]
        cases = sorted(k for g, k in at if g in emitted)
        assert cases == list(range(1, 255)), f"{mv.POSITION_NAMES[p]}: {254 - len(cases)} non-empty cases not emitted"
    print(f"atlas: all 254 non-empty cases emitted at {', '.join(mv.POSITION_NAMES)}; {len(ref['tri'])} triangles")


def test_boundary_values(built):
    xyz, vox = mv.boundary_values()
    three_way(xyz, vox)


def test_seams_and_key_range(built):
    xyz, vox = mv.seams_and_keys()
    (x, _, t), ref = three_way(xyz, vox)
    assert ref["n_edges"] > len(x)                                       # seam cubes next to a missing block drop vertices
    hi = (ref["cube"] // 8 == mv.KEY_HI).any(1)
    assert hi.any() and not ((ref["cube"] // 8 == mv.KEY_HI) & (ref["cube"] % 8 == 7)).any()


@pytest.mark.parametrize("name", ["sphere", "gyroid"])
def test_closed_fields(built, name):
    xyz, vox = getattr(mv, name)()
    (x, _, t), _ = three_way(xyz, vox)
    t = t.astype(np.int64)
    de = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    k = de[:, 0] << 32 | de[:, 1]
    assert len(np.unique(k)) == len(k), "a directed edge appears twice"
    assert np.isin(de[:, 1] << 32 | de[:, 0], k).all(), "an edge without its reverse: the mesh is open"
    P = x.astype(np.float64)
    nrm = np.cross(P[t[:, 1]] - P[t[:, 0]], P[t[:, 2]] - P[t[:, 0]])
    grad = getattr(mv, name + "_grad")(P[t].mean(1) / float(mv.VS))
    facing = (nrm * grad).sum(1)
    assert (facing > 0).all(), f"{int((facing <= 0).sum())} of {len(t)} faces do not point to sdf > 0"
    if name == "sphere":
        E = np.unique(np.sort(de, 1), axis=0)
        assert len(x) - len(E) + len(t) == 2


@pytest.mark.parametrize("name", ["no_crossing", "all_unusable"])
def test_degenerate_volumes(built, name):
    xyz, vox = getattr(mv, name)()
    (x, c, t), _ = three_way(xyz, vox)
    assert len(xyz) and len(x) == 0 and len(c) == 0 and len(t) == 0


def test_three_level_scans(built):
    xyz, vox = mv.large()
    assert len(xyz) * 512 > 2048 ** 2 * 2
    (x, _, t), _ = three_way(xyz, vox)
    assert len(t) > 100000


def frames():
    return synth.make_frames(6, seed=13, width=160, height=120, loop_frames=300)


def test_round_trip_restores_the_volume(built):
    D, C, P, K = frames()
    p = params(width=160, height=120, batch_frames=4)
    a = tsdf.TsdfVolume(p, device=0)
    a.integrate_batch(D[:3], C[:3], P[:3], K); a.sync()
    xa, va = a.download_blocks(sort=False)                              # heap order: upload must not depend on it
    b = tsdf.TsdfVolume(p, device=0)
    b.upload_blocks(xa, va)
    assert same_bytes(b.download_blocks(), a.download_blocks()), "download after upload differs"
    assert same_bytes(b.extract_mesh(), a.extract_mesh()), "mesh of the restored volume differs"
    for v in (a, b):
        v.integrate_batch(D[3:], C[3:], P[3:], K); v.sync()
    ga, gb = a.download_blocks(), b.download_blocks()
    assert same_bytes(ga, gb), "integration into the restored volume differs"
    o = ob.OracleTsdf(p)
    for i in range(len(D)):
        o.integrate(D[i], C[i], P[i], K)
    assert same_bytes(ga, o.export()), "volume differs from the oracle fused directly"
    assert a.stats().blocks_allocated == b.stats().blocks_allocated == len(ga[0])
    assert same_bytes(b.extract_mesh(), o.extract_mesh())
    # reset after an upload leaves an empty volume, and the next integration starts from zero
    b.reset()
    assert b.stats().blocks_allocated == 0 and len(b.download_blocks()[0]) == 0 and len(b.extract_mesh()[2]) == 0
    b.integrate_batch(D[:3], C[:3], P[:3], K); b.sync()
    assert same_bytes(b.download_blocks(), (xa[np.argsort(mr.pack(xa))], va[np.argsort(mr.pack(xa))]))
    a.close(); b.close(); o.close()


def test_upload_refusals_leave_the_volume(built):
    xyz, vox = mv.seams_and_keys()
    vol = tsdf.TsdfVolume(params(max_blocks=len(xyz) + 4, hash_slots=256), device=0)
    vol.upload_blocks(xyz[:20], vox[:20])
    before = vol.download_blocks()
    big = np.array([[x, 100, 100] for x in range(len(xyz) - 20 + 5)], np.int32)      # one block more than the heap has left
    bad = [(np.array([[1 << 20, 0, 0]]), vox[:1], ERR_ARG),                           # outside the key range
           (np.array([[0, 0, -(1 << 20) - 1]]), vox[:1], ERR_ARG),
           (np.concatenate([xyz[20:22], xyz[21:22]]), vox[20:23], ERR_ARG),            # given twice
           (xyz[19:21], vox[19:21], ERR_ARG),                                          # already present
           (big, np.zeros((len(big), 512), tsdf.VOXEL_DTYPE), ERR_CAPACITY)]
    for bx, bv, code in bad:
        with pytest.raises(ScnError) as e:
            vol.upload_blocks(bx, bv)
        assert e.value.code == code
        assert same_bytes(vol.download_blocks(), before) and vol.stats().blocks_allocated == 20
    vol.upload_blocks(xyz[20:], vox[20:])
    assert same_bytes(vol.extract_mesh(), gpu_mesh(xyz, vox))
    vol.close()
