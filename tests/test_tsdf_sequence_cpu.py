"""The TSDF spec over several frames, on the CPU: a volume fused frame after frame by the scalar oracle (oracle/tsdf_oracle.c)
must be the float64 fusion of tests/tsdf_reference.py (fuse_sequence): the running weighted mean of the sdf, the integer
weight capped at weight_max (and the capped weight used by the next update), the colour rounded to the nearest byte, and
updates only in blocks the frame's own walk touched.

The single-frame checks never see a second update of a voxel, and the GPU kernels are pinned to the oracle bit for bit, so a
mistake in the averaging shared by both would pass every other test.  The negative controls at the end fuse the reference's
own per-frame samples with numpy, once as the spec says and once with one such mistake each, and show that check_sequence
tells them apart."""
import numpy as np
import pytest

import oracle_bindings as ob
import tsdf_reference as tref
from scannet_b200 import synth
from test_tsdf_reference_cpu import mirrored, params, plane_frame, rescaled_depth, translated


def tint(c, i):
    """Per-frame colour that varies across the image: voxel colour averages land between bytes, so rounding shows."""
    H, W = c.shape[:2]
    pat = (np.arange(W)[None, :] * 7 + np.arange(H)[:, None] * 3 + 41 * i) % 61
    return ((c.astype(np.int64) + pat[..., None] * np.array([1, 2, 3])) % 256).astype(np.uint8)


def room_seq(n, W=24, H=18, loop=1200, colour="on", invalid=(), zoom=6.0, seed=31, centre=(3.0, 2.5, 1.5)):
    """n frames of the box room's camera loop through a lens `zoom` times longer than the default (a few thousand blocks),
    with the world moved so that `centre` is its origin (small coordinates keep the float32 margins, and so the share of
    ambiguous voxels, small); colour "on", "off" or "alternate" (every other frame depth-only); frames whose index is in
    `invalid` get the all -inf pose (skipped)."""
    sc = synth.BoxRoomScene(seed=seed, width=W, height=H, fx=zoom * synth.FX * W / 640.0, fy=zoom * synth.FY * H / 480.0,
                            cx=(W - 1) / 2.0, cy=(H - 1) / 2.0)
    K = sc.intrinsics()
    out = []
    for j in range(n):
        T = sc.camera_pose(j, loop)
        d, c = sc.render(T)
        T = T.copy(); T[:3, 3] -= np.asarray(centre, np.float32)
        c = tint(c, j)
        if colour == "off" or (colour == "alternate" and j % 2):
            c = None
        if j in invalid:
            T = np.full((4, 4), -np.inf, np.float32)
        out.append((d, c, T, K))
    return out


def receding_plane(dists, z_plane=2.0, W=64, H=48):
    """Identity-oriented camera backing away from the plane z = z_plane: with max_integration_distance below the far
    distances, the late frames walk no pixel (d >= max_integration_distance) while their depth, still inside
    [depth_min, depth_max], covers the blocks the early frames allocated - which they must leave alone."""
    out = []
    for j, dist in enumerate(dists):
        d, c, T, K = plane_frame(W, H, raw=int(round(dist * 1000)))
        T = T.copy(); T[2, 3] = z_plane - dist
        out.append((d, tint(c, j), T, K))
    return out


SEQS = {
    "room_8_colour": (lambda: room_seq(8), {}),
    "room_40_alternating": (lambda: room_seq(40, loop=4000, colour="alternate"), {}),
    "room_12_ws2_depth_only": (lambda: room_seq(12, colour="off"), {"weight_sample": 2}),
    "room_10_ws10_wmax40": (lambda: room_seq(10, colour="alternate"), {"weight_sample": 10, "weight_max": 40}),
    "room_4_ws1000": (lambda: room_seq(4), {"weight_sample": 1000}),
    "room_10_wmax1": (lambda: room_seq(10), {"weight_max": 1}),
    "room_10_wmax2_alternating": (lambda: room_seq(10, colour="alternate"), {"weight_max": 2}),
    "room_6_invalid_poses": (lambda: room_seq(6, invalid=(1, 2, 4)), {}),
    "plane_close_ws171": (lambda: [(d, tint(c, j), T, K) for j, (d, c, T, K) in enumerate([plane_frame(48, 36, raw=110)] * 5)],
                          {"weight_sample": 171, "voxel_size": 2.0 ** -9}),
    "plane_close_ws172": (lambda: [(d, tint(c, j), T, K) for j, (d, c, T, K) in enumerate([plane_frame(48, 36, raw=110)] * 5)],
                          {"weight_sample": 172, "voxel_size": 2.0 ** -9}),
    "receding_plane": (lambda: receding_plane([0.8, 1.0, 1.2, 1.6, 1.9, 2.2]),
                       {"voxel_size": 2.0 ** -8, "max_integration_distance": 1.5}),
    "mirrored_6": (lambda: [mirrored(f) for f in room_seq(6)], {}),
    "translated_6": (lambda: [translated(f, (-9.5, -7.25, -4.0)) for f in room_seq(6, colour="alternate")], {}),
    "rescaled_depth_6": (lambda: [rescaled_depth(f, 5000.0) for f in room_seq(6)], {"depth_shift": 5000.0}),
}


@pytest.fixture(scope="module")
def oracle_lib():
    try:
        return ob.tsdf_oracle_lib()
    except FileNotFoundError as e:
        pytest.skip(str(e))


def fuse_oracle(p, frames, metres=False):
    o = ob.OracleTsdf(p, threads=4)
    for d, c, T, K in frames:
        (o.integrate_metres if metres else o.integrate)(d, c, T, K)
    xyz, vox = o.export()
    mesh = o.extract_mesh()
    o.close()
    return xyz, vox, mesh


def case(name):
    make, over = SEQS[name]
    frames = make()
    d = frames[0][0]
    return params(d.shape[1], d.shape[0], **over), frames


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", sorted(SEQS))
def test_oracle_sequence_is_float64_fusion(oracle_lib, name):
    p, frames = case(name)
    xyz, vox, (mx, _, mt) = fuse_oracle(p, frames)
    assert len(xyz) > 0
    # with weight_sample 1000, w1 = floor(1500 (1 - dz)) differs between neighbouring pixels: a voxel next to a pixel-rounding
    # boundary is then ambiguous whatever the depths
    ref = tref.check_sequence(p, frames, xyz, vox, max_ambiguous=0.1 if p.weight_sample >= 1000 else 0.05)
    assert ref["frames"] == sum(np.asarray(T)[0, 0] != -np.inf for _, _, T, _ in frames)
    assert len(mt) > 0
    tref.check_mesh(p, xyz, vox, mx, mt)
    if p.weight_max < 255 or p.weight_sample >= 171:
        assert vox["w"].max() == min(p.weight_max, 255)                 # the cap is reached: later updates average against it


def test_receding_camera_leaves_untouched_blocks_alone(oracle_lib):
    """The late frames of the receding case update no allocated block, although each block's voxels project onto valid
    depth: only the walk's touched set keeps them out."""
    p, frames = case("receding_plane")
    xyz, vox, _ = fuse_oracle(p, frames)
    ups = list(tref.frame_updates(p, frames, xyz))
    late = ups[-1]
    assert not late["in_possible"].any() and late["upd"].sum() > 1000


def test_metres_input_matches_raw(oracle_lib):
    """Depth handed over in metres (the bilateral filter's output) is taken exactly: the float64 fusion of the same frames
    in metres accepts the oracle's metres path."""
    p, frames = case("room_8_colour")
    fm = [(np.where(d == 0, -np.inf, d.astype(np.float32) / np.float32(1000.0)).astype(np.float32), c, T, K)
          for d, c, T, K in frames]
    xyz, vox, _ = fuse_oracle(p, fm, metres=True)
    tref.check_sequence(p, fm, xyz, vox)


# ---- negative controls: the reference's own samples fused in numpy binary32, as the spec says and with one mistake each
def numpy_fuse(p, frames, xyz, mistake=None):
    """Voxels in the oracle's export layout from fuse_sequence's per-frame samples (tref.frame_updates), with the spec's
    update in binary32: sdf' = (sdf0 w0 + s w1) / (w0 + w1), w' = min(w0 + w1, weight_max), colour floor(avg + 1/2)."""
    n = len(xyz)
    sdf = np.zeros((n, 512), np.float32); w = np.zeros((n, 512), np.int64); w_sum = np.zeros((n, 512), np.int64)
    col = np.zeros((n, 512, 3), np.int64)
    f32 = np.float32
    for fr in tref.frame_updates(p, frames, xyz):
        u = fr["upd"] & (True if mistake == "every_block_touched" else fr["in_possible"])
        w0 = w_sum if mistake == "uncapped_w0" else w
        w1 = fr["w1"]
        ws = w0 + w1
        inv = (f32(1.0) / np.maximum(ws + (1 if mistake == "rcp_plus_one" else 0), 1).astype(f32)).astype(f32)
        sn = (sdf * w0.astype(f32) + fr["sdf"].astype(f32) * w1.astype(f32)) * inv
        if fr["has_rgb"]:
            q = (col * w0[..., None] + fr["rgb"].astype(np.int64) * w1[..., None]).astype(f32) * inv[..., None]
            cn = np.floor(q if mistake == "truncated_colour" else q + f32(0.5)).astype(np.int64)
            col = np.where(u[..., None], cn, col)
        sdf = np.where(u, sn, sdf).astype(f32)
        w_sum = np.where(u, ws, w_sum)
        w = np.where(u, np.minimum(ws, int(p.weight_max)), w)
    vox = np.zeros((n, 512), ob.VOXEL_DTYPE)
    vox["sdf"] = sdf; vox["w"] = w
    vox["r"], vox["g"], vox["b"] = col[..., 0], col[..., 1], col[..., 2]
    return vox


CONTROLS = [
    ("rcp_plus_one", "room_10_wmax2_alternating", "sdf"),
    ("uncapped_w0", "room_10_wmax2_alternating", "sdf"),
    ("truncated_colour", "room_8_colour", "colour"),
    ("every_block_touched", "receding_plane", "weights"),
]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("mistake,name,what", CONTROLS)
def test_check_sequence_rejects_a_mistaken_fusion(oracle_lib, mistake, name, what):
    p, frames = case(name)
    xyz, _, _ = fuse_oracle(p, frames)
    tref.check_sequence(p, frames, xyz, numpy_fuse(p, frames, xyz))            # the spec, restated in numpy: accepted
    with pytest.raises(AssertionError, match=what):
        tref.check_sequence(p, frames, xyz, numpy_fuse(p, frames, xyz, mistake))


def test_oracle_bilateral_is_float64_filter(oracle_lib):
    """The oracle's statement of the depth pre-filter against the float64 one (tests/tsdf_reference.py:bilateral_f64)."""
    from scannet_b200 import synth
    for sd, sr, (W, H) in [(2.0, 0.05, (97, 61)), (4.0, 0.05, (80, 60)), (0.1, 0.05, (80, 60))]:
        D, _, _, _ = synth.make_frames(1, seed=5, width=W, height=H, noise_mm=4.0, drop=0.08, with_color=False)
        ref, taps = tref.bilateral_f64(D[0], 1000.0, sd, sr)
        o = ob.oracle_bilateral(D[0], 1000.0, sd, sr)
        inv = np.isinf(ref)
        assert (np.isinf(o) == inv).all()
        assert np.abs(o[~inv] - ref[~inv]).max() <= (2 * taps + 8) * 2.0 ** -24 * np.abs(ref[~inv]).max()
