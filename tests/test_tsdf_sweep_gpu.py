"""TSDF fusion and marching cubes on the GPU, bit for bit against oracle/tsdf_oracle.c, across the parameter space the other
tests leave out: per-sample weights past the 512-entry reciprocal table, the saturated-weight hot path, sub-millimetre to
10 cm voxels (the k_alloc window / shared-map / step-cap fallbacks), camera jumps, negative and key-limit coordinates, mirrored
and axis-aligned cameras, degenerate and maximal frame shapes, the ends of the depth range, frame grouping and CTA
reservation, exact capacity, and the bilateral filter's radius limits.

Every case compares the block set, the voxel bytes, N_u, N_b, the skipped-frame count and the mesh (vertex bits, colours,
triangle order).  Single-frame cases are also checked against the float64 statement of fusion (tests/tsdf_reference.py)."""
import numpy as np
import pytest

import oracle_bindings as ob
import tsdf_reference as tref
from scannet_b200 import ScnError, synth, tsdf
from test_tsdf_reference_cpu import mirrored, plane_frame, translated

pytestmark = pytest.mark.gpu

ERR_CAPACITY = -5


def room(n, W=64, H=48, loop=120, seed=41, offset=None, jump=None):
    """n frames of the box room (depth u16, rgb, poses, K); `offset` translates the world, `jump` adds a translation to
    every other pose (the same view seen from far away)."""
    D, C, P, K = synth.make_frames(n, seed=seed, width=W, height=H, loop_frames=loop)
    if offset is not None:
        P[:, :3, 3] += np.asarray(offset, np.float32)
    if jump is not None:
        P[1::2, :3, 3] += np.asarray(jump, np.float32)
    return D, C, P, K


def stack(frame, n=1):
    d, c, T, K = frame
    return np.stack([d] * n), np.stack([c] * n), np.stack([T] * n), K


def prm(W, H, **kw):
    kw.setdefault("max_blocks", 1 << 17)
    kw.setdefault("hash_slots", 1 << 19)
    return tsdf.default_params(width=W, height=H, **kw)


def run_gpu(p, D, C, P, K, api="batch", mesh=True):
    vol = tsdf.TsdfVolume(p, device=0)
    try:
        if api == "batch":
            vol.integrate_batch(D, C, P, K)
        elif api == "single":
            for i in range(len(D)):
                vol.integrate(D[i], None if C is None else C[i], P[i], K)
        else:
            import torch
            d = torch.from_numpy(np.ascontiguousarray(D).view(np.int16)).cuda()
            c = None if C is None else torch.from_numpy(np.ascontiguousarray(C)).cuda()
            vol.integrate_device(len(D), d.data_ptr(), None if c is None else c.data_ptr(), P, K)
        vol.sync()
        gx, gv = vol.download_blocks()
        st = vol.stats()
        m = vol.extract_mesh() if mesh else None
    finally:
        vol.close()
    return gx, gv, st, m


def run_oracle(p, D, C, P, K, mesh=True):
    o = ob.OracleTsdf(p, threads=8)
    for i in range(len(D)):
        o.integrate(D[i], None if C is None else C[i], P[i], K)
    ox, ov = o.export()
    oc = o.counters()
    m = o.extract_mesh() if mesh else None
    o.close()
    return ox, ov, oc, m


def compare(p, D, C, P, K, api="batch", mesh=True, reference=True, max_ambiguous=0.02):
    """GPU vs oracle, zero tolerance; one valid frame: also the float64 checks.  Returns the oracle's result."""
    gx, gv, st, gm = run_gpu(p, D, C, P, K, api, mesh)
    ox, ov, oc, om = run_oracle(p, D, C, P, K, mesh)
    assert gx.shape == ox.shape and (gx == ox).all(), f"block sets differ ({len(gx)} vs {len(ox)})"
    same = (gv.view(np.uint64) == ov.view(np.uint64))
    assert same.all(), (f"{int((~same).sum())} voxels differ; max |dsdf| {np.abs(gv['sdf'] - ov['sdf']).max():.3g}, "
                        f"weights {np.unique(gv['w'][~same])[:8]} vs {np.unique(ov['w'][~same])[:8]}")
    assert st.voxels_updated == oc["total_updated"] and st.blocks_visited == oc["total_touched"]
    assert st.frames_integrated == oc["frames_done"] and st.frames_skipped == oc["frames_skipped"]
    if mesh:
        (gxyz, grgb, gtri), (oxyz, orgb, otri) = gm, om
        assert gxyz.shape == oxyz.shape and gxyz.tobytes() == oxyz.tobytes(), "mesh vertices differ"
        assert grgb.tobytes() == orgb.tobytes() and gtri.shape == otri.shape and (gtri == otri).all(), "mesh colours / triangles differ"
    if reference and oc["frames_done"] == 1 and len(gx):
        k = int(np.nonzero(P[:, 0, 0] != -np.inf)[0][0])
        tref.check_single_frame(p, D[k], None if C is None else C[k], P[k], K, gx, gv, max_ambiguous)
        tref.check_allocation(p, D[k], P[k], K, gx)
        if mesh:
            tref.check_mesh(p, gx, gv, gm[0], gm[2])
    return ox, ov, oc


# ---- per-sample weight ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("color", [False, True])
@pytest.mark.parametrize("ws", [0, 1, 2, 1000])
def test_weight_sample_room(built, ws, color):
    D, C, P, K = room(4)
    compare(prm(64, 48, weight_sample=ws, batch_frames=4), D, C if color else None, P, K)


@pytest.mark.parametrize("color", [False, True])
def test_weight_sample_1000_single_frame_float64(built, color):
    """w1 reaches 1500: every update takes the reciprocal past the 512-entry table"""
    D, C, P, K = room(1, W=80, H=60)
    compare(prm(80, 60, weight_sample=1000), D, C if color else None, P, K)


@pytest.mark.parametrize("color", [False, True])
@pytest.mark.parametrize("ws", [171, 172])
def test_weight_sample_close_plane(built, ws, color):
    """A fronto-parallel plane at 0.11 m: w1 = 256 (171) or 257 (172), so from the second frame on w0 + w1 is 511 or 512"""
    d, c, T, K = plane_frame(W=48, H=36, raw=110)
    D, C, P, _ = stack((d, c, T, K), 5)
    _, ov, _ = compare(prm(48, 36, weight_sample=ws, voxel_size=2.0 ** -9, batch_frames=8), D, C if color else None, P, K)
    assert ov["w"].max() == 255


@pytest.mark.timeout(300)
@pytest.mark.parametrize("api", ["batch", "device"])
@pytest.mark.parametrize("wmax", [1, 2, 3])
def test_saturated_weight_hot_path(built, wmax, api):
    """constant sample weight, depth only, batch 32: the weight counter runs far past weight_max within a batch"""
    D, _, P, K = room(44, loop=400)
    _, ov, _ = compare(prm(64, 48, weight_max=wmax, batch_frames=32), D, None, P, K, api=api)
    assert ov["w"].max() == wmax


# ---- voxel size -------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
def test_half_millimetre_voxels_leave_the_alloc_window(built):
    """0.5 mm voxels: rays reach blocks more than 511 cells from the camera block (the global-coordinate walk), the shared map
    overflows, and long walks hit the 48-step cap.  ~310 k blocks, 1.3 GB of heap."""
    D, C, P, K = room(3, loop=300)
    p = prm(64, 48, voxel_size=0.0005, max_blocks=360_000, hash_slots=1 << 20, batch_frames=4)
    ox, _, _ = compare(p, D, None, P, K, mesh=False)
    cam = np.floor(P[:, :3, 3] / (8 * 0.0005) + 1.0 / 16).astype(np.int64)
    far = np.abs(ox[:, None, :] - cam[None]).max(2).min(1).max()
    assert far > 511, far


@pytest.mark.parametrize("vs", [0.001, 0.02, 0.1])
def test_voxel_sizes(built, vs):
    D, C, P, K = room(3, loop=300)
    compare(prm(64, 48, voxel_size=vs, max_blocks=1 << 18, hash_slots=1 << 20), D, C, P, K)


# ---- poses ------------------------------------------------------------------------------------------------------------
def test_camera_jump_inside_an_allocation_group(built):
    """every other frame 25 m away: the window origin comes from the group's first frame"""
    D, C, P, K = room(8, jump=(25.0, -3.0, 1.0))
    compare(prm(64, 48, batch_frames=8), D, C, P, K)


def test_negative_world_coordinates(built):
    D, C, P, K = room(4, offset=(-20.0, -13.5, -7.25))
    compare(prm(64, 48), D, C, P, K)


@pytest.mark.parametrize("offset", [(33554.432 - 5.0, -33554.432 - 2.5, 0.0), (-33554.432 - 3.0, 0.0, 33554.432 - 1.5)])
def test_blocks_straddle_the_key_limit(built, offset):
    """4 mm voxels: block 2^20 starts at 33554.432 m; blocks at or beyond +-2^20 are dropped (k_alloc key_ok, and the
    marching-cubes neighbour lookup of a block that cannot exist)"""
    D, C, P, K = room(3, offset=offset)
    ox, _, _ = compare(prm(64, 48), D, C, P, K, reference=False)
    assert len(ox) and ((ox.max(0) == (1 << 20) - 1) | (ox.min(0) == -(1 << 20))).any()


def test_axis_aligned_identity_pose_single_frame(built):
    D, C, P, K = stack(plane_frame())
    compare(prm(64, 48, voxel_size=2.0 ** -8), D, C, P, K)


@pytest.mark.parametrize("n", [1, 3])
def test_mirrored_camera(built, n):
    D, C, P, K = room(n)
    f = [mirrored((D[i], C[i], P[i], K)) for i in range(n)]
    compare(prm(64, 48), np.stack([x[0] for x in f]), np.stack([x[1] for x in f]), np.stack([x[2] for x in f]), f[0][3])


def test_negative_world_single_frame_float64(built):
    D, C, P, K = stack(translated(plane_frame(), (-3.25, -1.5, -2.0)))
    compare(prm(64, 48, voxel_size=2.0 ** -8), D, C, P, K)


# ---- frame shapes -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wh", [(1, 1), (2, 3), (3, 2), (1, 37), (37, 1), (17, 16), (16, 17)])
def test_small_and_ragged_frames(built, wh):
    W, H = wh
    D, C, P, K = room(3, W=W, H=H)
    compare(prm(W, H, batch_frames=2), D, C, P, K)
    compare(prm(W, H, batch_frames=3), D[:1], C[:1], P[:1], K)


@pytest.mark.timeout(600)
def test_largest_frame(built):
    """2048 x 2048 = 2^22 pixels, the largest frame accepted"""
    D, _, P, K = room(1, W=2048, H=2048)
    compare(prm(2048, 2048, batch_frames=1, max_blocks=1 << 18, hash_slots=1 << 20), D, None, P, K, mesh=False, reference=False)


@pytest.mark.parametrize("wh", [(2048, 2049), (2394, 1752)])
def test_refused_frame_sizes(built, wh):
    with pytest.raises(ScnError):
        tsdf.TsdfVolume(prm(*wh, max_blocks=64, hash_slots=256, batch_frames=1), device=0)


def test_weight_sample_domain(built):
    with pytest.raises(ScnError):
        tsdf.TsdfVolume(prm(64, 48, weight_sample=(1 << 24) + 1), device=0)
    tsdf.TsdfVolume(prm(64, 48, weight_sample=1 << 24), device=0).close()


# ---- depth range ------------------------------------------------------------------------------------------------------
def depth_bands(raws, W=60, H=40):
    """Identity pose facing fronto-parallel planes: one vertical band of the image per raw depth value"""
    d, c, T, K = plane_frame(W, H)
    d = np.zeros((H, W), np.uint16)
    for i, r in enumerate(raws):
        d[:, i * W // len(raws):(i + 1) * W // len(raws)] = r
    K = K.copy(); K[0, 0] = K[1, 1] = 40.0
    return d, c, T, K


@pytest.mark.parametrize("maxint", [4.0, 0.05, 8.0])
@pytest.mark.parametrize("n", [1, 2])
def test_depth_at_range_ends(built, maxint, n):
    """depth exactly at depth_min, depth_max and max_integration_distance, and just outside"""
    D, C, P, K = stack(depth_bands([99, 100, 101, 3999, 4000, 4001, 5999, 6000, 6001]), n)
    # voxels reading the bands exactly at depth_min / depth_max are ambiguous for the float64 check
    ox, _, _ = compare(prm(60, 40, max_integration_distance=maxint, voxel_size=0.02), D, C, P, K, max_ambiguous=0.7)
    if maxint < 0.1:
        assert len(ox) == 0


def test_depth_shift(built):
    D, C, P, K = room(3)
    D = np.round(D.astype(np.float64) * 5.0).astype(np.uint16)
    compare(prm(64, 48, depth_shift=5000.0), D, C, P, K)
    compare(prm(64, 48, depth_shift=5000.0), D[:1], C[:1], P[:1], K)


# ---- scheduling -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", [1, 2, 7, 32])
def test_frame_grouping(built, batch):
    """one k_alloc CTA walks 4 frames of a batch: batches below one group, a partial last group (7 = 4 + 3) and 8 groups"""
    D, C, P, K = room(35, loop=200)
    compare(prm(64, 48, batch_frames=batch), D, None, P, K, mesh=batch == 7)


# ---- capacity ---------------------------------------------------------------------------------------------------------
def test_exact_capacity_and_minimum_hash_table(built):
    D, C, P, K = room(3)
    ox, _, _ = compare(prm(64, 48), D, C, P, K)
    n = len(ox)
    compare(prm(64, 48, max_blocks=n, hash_slots=1), D, C, P, K)          # table of 2*max_blocks slots (rounded up)
    vol = tsdf.TsdfVolume(prm(64, 48, max_blocks=n - 1, hash_slots=1), device=0)
    try:
        vol.integrate_batch(D, C, P, K)
        with pytest.raises(ScnError) as e:
            vol.sync()
        assert e.value.code == ERR_CAPACITY
    finally:
        vol.close()


# ---- bilateral filter -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sd", [4.0, 0.1])
def test_bilateral_radius_limits(built, sd):
    D, _, _, _ = synth.make_frames(1, seed=5, width=80, height=60, noise_mm=4.0, drop=0.08, with_color=False)
    g = tsdf.bilateral_filter(D[0], 1000.0, sd, 0.05)
    o = ob.oracle_bilateral(D[0], 1000.0, sd, 0.05)
    inv = np.isinf(o)
    assert (np.isinf(g) == inv).all()
    assert (np.abs(g[~inv] - o[~inv]) / np.abs(o[~inv])).max() < 2e-6


def test_bilateral_radius_above_limit_is_refused(built):
    D, _, _, _ = synth.make_frames(1, seed=5, width=32, height=24, with_color=False)
    with pytest.raises(ScnError):
        tsdf.bilateral_filter(D[0], 1000.0, 4.01, 0.05)
