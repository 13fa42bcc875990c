"""The TSDF spec itself against geometry, on the CPU: one frame fused by the scalar oracle (oracle/tsdf_oracle.c) must be
the float64 statement of projective TSDF fusion in tests/tsdf_reference.py - updated voxels, sdf to ~1e-5 m, exact weights and
colours - its block set must cover the truncation band, and its marching-cubes vertices must sit at the zero crossings.

The GPU kernels are pinned to the oracle bit for bit elsewhere; a convention mistake shared by both (half a pixel, a transposed
pose, voxel corner for centre) would pass those tests and fails these."""
import numpy as np
import pytest

import oracle_bindings as ob
import tsdf_reference as tref
from scannet_b200 import synth
from scannet_b200._lib import TsdfParams


def params(w, h, **kw):
    p = TsdfParams(); p.voxel_size = 0.004; p.trunc_base = 0.02; p.trunc_scale = 0.01; p.depth_min = 0.1; p.depth_max = 6.0
    p.max_integration_distance = 4.0; p.weight_sample = 1; p.weight_max = 255; p.width = w; p.height = h; p.depth_shift = 1000.0
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def room_frame(i, W=96, H=72, loop=24, seed=31, cx=None, cy=None):
    """Frame i of the synthetic box room's camera loop: (depth u16 [H,W], rgb [H,W,3], cam2world, K)."""
    sc = synth.BoxRoomScene(seed=seed, width=W, height=H, fx=synth.FX * W / 640.0, fy=synth.FY * H / 480.0,
                            cx=(W - 1) / 2.0 if cx is None else cx, cy=(H - 1) / 2.0 if cy is None else cy)
    T = sc.camera_pose(i, loop)
    d, c = sc.render(T)
    return d, c, T, sc.intrinsics()


def plane_frame(W=64, H=48, raw=1000):
    """Identity pose facing the plane z = 1 m with fx = fy = 128 and an integer principal point: with 2^-8 m voxels the voxels
    of the plane project exactly onto pixel centres and half-pixels (round half to even), the centre row and column are rays
    parallel to the axes, and the plane's voxel layer has sdf exactly 0."""
    K = np.eye(4, dtype=np.float32); K[0, 0] = K[1, 1] = 128.0; K[0, 2] = W // 2; K[1, 2] = H // 2
    D = np.full((H, W), raw, np.uint16)
    C = np.zeros((H, W, 3), np.uint8); C[..., 0] = np.arange(W)[None] * 3; C[..., 1] = np.arange(H)[:, None] * 5; C[..., 2] = 77
    return D, C, np.eye(4, dtype=np.float32), K


def mirrored(frame):
    """The same view through a camera with negative fx: columns reversed, cx' = W - 1 - cx."""
    d, c, T, K = frame
    K = K.copy(); W = d.shape[1]
    K[0, 0] = -K[0, 0]; K[0, 2] = W - 1 - K[0, 2]
    return np.ascontiguousarray(d[:, ::-1]), np.ascontiguousarray(c[:, ::-1]), T, K


def translated(frame, off):
    d, c, T, K = frame
    T = T.copy(); T[:3, 3] += np.asarray(off, np.float32)
    return d, c, T, K


def rescaled_depth(frame, shift):
    d, c, T, K = frame
    return np.round(d.astype(np.float64) * shift / 1000.0).astype(np.uint16), c, T, K


CASES = {
    "room_pose0": (lambda: room_frame(0), {}),
    "room_pose7": (lambda: room_frame(7), {}),
    "room_pose15_depth_only": (lambda: room_frame(15), {"_no_color": True}),
    "plane_half_pixels": (lambda: plane_frame(), {"voxel_size": 2.0 ** -8}),
    "principal_point_outside": (lambda: room_frame(3, cx=-20.0, cy=90.0), {}),
    "weight_sample_10": (lambda: room_frame(5), {"weight_sample": 10, "weight_max": 40}),
    "weight_sample_1000": (lambda: room_frame(9), {"weight_sample": 1000}),
    "trunc_scale_0": (lambda: room_frame(11), {"trunc_scale": 0.0}),
    "depth_shift_5000": (lambda: rescaled_depth(room_frame(13), 5000.0), {"depth_shift": 5000.0}),
    "negative_world": (lambda: translated(room_frame(17), (-9.5, -7.25, -4.0)), {}),
    "mirrored_camera": (lambda: mirrored(room_frame(19)), {}),
}


@pytest.fixture(scope="module")
def oracle_lib():
    try:
        return ob.tsdf_oracle_lib()
    except FileNotFoundError as e:
        pytest.skip(str(e))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_single_frame_is_float64_fusion(oracle_lib, name):
    make, over = CASES[name]
    over = dict(over)
    no_color = over.pop("_no_color", False)
    D, C, T, K = make()
    C = None if no_color else C
    p = params(D.shape[1], D.shape[0], **over)
    o = ob.OracleTsdf(p, threads=4)
    o.integrate(D, C, T, K)
    xyz, vox = o.export()
    assert len(xyz) > 0
    tref.check_single_frame(p, D, C, T, K, xyz, vox)
    tref.check_allocation(p, D, T, K, xyz)
    mx, _, mt = o.extract_mesh()
    assert len(mt) > 0
    tref.check_mesh(p, xyz, vox, mx, mt)
    o.close()


def test_plane_case_pins_half_pixel_rounding_and_zero_sdf(oracle_lib):
    """The dyadic plane really lands on the edges it is meant to reach."""
    D, C, T, K = plane_frame()
    p = params(D.shape[1], D.shape[0], voxel_size=2.0 ** -8)
    o = ob.OracleTsdf(p, threads=2)
    o.integrate(D, C, T, K)
    xyz, vox = o.export()
    ref = tref.fuse_single_frame(p, D, C, T, K, xyz)
    on_plane = (vox["w"] > 0) & (vox["sdf"] == 0.0)
    assert on_plane.sum() >= 0.9 * D.size                      # one voxel layer with sdf exactly 0
    g = 8 * xyz[:, None, 0] + (np.arange(512)[None] & 7)
    half = on_plane & (g % 2 == 1)                             # u = g/2 + cx: exactly half a pixel
    assert half.sum() > 100 and not ref["amb"][half].any()
    # round half to even: voxel 2k+1 of the plane reads pixel cx + k (k even) or cx + k + 1 (k odd) - its colour says which
    col = (vox["r"][half].astype(int)) // 3
    k = (g[half] - 1) // 2
    assert (col == np.where(k % 2 == 0, k, k + 1) + K[0, 2]).all()
    o.close()


def test_reference_rejects_a_half_pixel_shift(oracle_lib):
    """The float64 check is sharp enough to see half a pixel: the oracle's volume, checked against a principal point moved
    by 0.5 px, fails."""
    D, C, T, K = room_frame(7)
    p = params(D.shape[1], D.shape[0])
    o = ob.OracleTsdf(p, threads=4)
    o.integrate(D, C, T, K)
    xyz, vox = o.export()
    K2 = K.copy(); K2[0, 2] += 0.5
    with pytest.raises(AssertionError):
        tref.check_single_frame(p, D, C, T, K2, xyz, vox)
    T2 = T.copy(); T2[:3, :3] = T[:3, :3].T                     # transposed rotation
    with pytest.raises(AssertionError):
        tref.check_single_frame(p, D, C, T2, K, xyz, vox)
    o.close()
