"""TSDF fusion on the GPU over several batches, against the oracle bit for bit AND against the float64 fusion of
tests/tsdf_reference.py (check_sequence) whatever the frame count: the running average, the weight cap and the capped weight
the next update uses, colour rounding, and updates only in blocks the frame's own walk touched.

Integrate instantiations reached (COLOR x CONSTW x STATS x {column, TMA} = 16), each by a case of at least two batches:
  * test_variant_matrix: all 16, one parameter set each (colour = rgb given, CONSTW = weight_sample 1, STATS = no NO_STATS
    flag, kernel forced by KERNEL_COLUMN / KERNEL_TMA);
  * test_mixed_colour_and_depth_only_calls: <1,1,1> and <0,1,1> (weight_sample 1), <1,0,1> and <0,0,1> (weight_sample 2):
    through integrate_batch / integrate_device on the column kernel (batches of 3) and the TMA kernel (each call's 1-frame
    tail), through integrate on the TMA kernel;
  * test_saturated_weight_hot_path, test_weight_reaches_255: <0,1,1> column (weight_max 1-3, 255);
  * test_bench_shape_sampled: <0,1,1> column, 640x480;
  * test_filtered_depth: k_alloc<1> with <1,1,1> on both kernels.
k_alloc<0> runs in every other case."""
import numpy as np
import pytest

import oracle_bindings as ob
import tsdf_reference as tref
from scannet_b200 import synth, tsdf
from test_tsdf_sequence_cpu import room_seq

pytestmark = pytest.mark.gpu


def prm(W, H, **kw):
    kw.setdefault("max_blocks", 1 << 17)
    kw.setdefault("hash_slots", 1 << 19)
    return tsdf.default_params(width=W, height=H, **kw)


def split(frames):
    D = np.stack([f[0] for f in frames])
    P = np.stack([np.asarray(f[2], np.float32) for f in frames])
    return D, P, frames[0][3]


def run_gpu(p, calls, api):
    """calls: list of frame lists, each handed over in one call (`batch`, `device`) or frame by frame (`single`); all frames
    of one call carry colour or none do."""
    import torch
    vol = tsdf.TsdfVolume(p, device=0)
    try:
        for frames in calls:
            D, P, K = split(frames)
            C = None if frames[0][1] is None else np.stack([f[1] for f in frames])
            if api == "batch":
                vol.integrate_batch(D, C, P, K)
            elif api == "single":
                for i in range(len(D)):
                    vol.integrate(D[i], None if C is None else C[i], P[i], K)
            else:
                d = torch.from_numpy(np.ascontiguousarray(D).view(np.int16)).cuda()
                c = None if C is None else torch.from_numpy(np.ascontiguousarray(C)).cuda()
                vol.integrate_device(len(D), d.data_ptr(), None if c is None else c.data_ptr(), P, K)
                torch.cuda.synchronize()
        vol.sync()
        gx, gv = vol.download_blocks()
        return gx, gv, vol.stats(), vol.extract_mesh()
    finally:
        vol.close()


_accepted = {}


def compare(p, calls, api="batch", metres=None, sample=None, max_ambiguous=0.05, min_exact_colour=0.8):
    """GPU vs oracle with zero tolerance (block set, voxel bytes, N_u / N_b with stats on, mesh), then check_sequence and
    check_mesh on the GPU volume.  `metres`: per-frame depth images in metres handed to the oracle and to the float64
    fusion instead of the raw depth (the pre-filtered path).  A volume byte-identical to one check_sequence has already
    accepted for the same parameters and frames is not checked again."""
    frames = [f for c in calls for f in c]
    gx, gv, st, (gxyz, grgb, gtri) = run_gpu(p, calls, api)
    ref_frames = frames if metres is None else [(m, c, T, K) for m, (_, c, T, K) in zip(metres, frames)]
    o = ob.OracleTsdf(p, threads=8)
    for d, c, T, K in ref_frames:
        (o.integrate if metres is None else o.integrate_metres)(d, c, T, K)
    ox, ov = o.export(); oc = o.counters(); oxyz, orgb, otri = o.extract_mesh(); o.close()
    assert gx.shape == ox.shape and (gx == ox).all(), f"block sets differ ({len(gx)} vs {len(ox)})"
    same = gv.view(np.uint64) == ov.view(np.uint64)
    assert same.all(), f"{int((~same).sum())} voxels differ from the oracle"
    assert st.frames_integrated == oc["frames_done"] and st.frames_skipped == oc["frames_skipped"]
    if not p.flags & tsdf.NO_STATS:
        assert st.voxels_updated == oc["total_updated"] and st.blocks_visited == oc["total_touched"]
    assert gxyz.tobytes() == oxyz.tobytes() and grgb.tobytes() == orgb.tobytes() and gtri.tobytes() == otri.tobytes(), "mesh differs"
    key = (bytes(p)[:44], sample, b"".join(np.ascontiguousarray(f[0]).tobytes() + np.asarray(f[2], np.float32).tobytes() +
                                           (b"-" if f[1] is None else np.ascontiguousarray(f[1]).tobytes()) for f in ref_frames))
    vb = gx.tobytes() + gv.tobytes()
    if _accepted.get(key) != vb:
        tref.check_sequence(p, ref_frames, gx, gv, max_ambiguous=max_ambiguous, min_exact_colour=min_exact_colour, sample=sample)
        tref.check_mesh(p, gx, gv, gxyz, gtri)
        _accepted[key] = vb
    return gv


# ---- the 16 integrate instantiations --------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("kernel", ["column", "tma"])
@pytest.mark.parametrize("stats", [True, False])
@pytest.mark.parametrize("ws", [1, 2])
@pytest.mark.parametrize("colour", [True, False])
def test_variant_matrix(built, colour, ws, stats, kernel):
    """12 frames in batches of 4 (3 batches: every block is stored and loaded again between batches)"""
    flags = (tsdf.KERNEL_COLUMN if kernel == "column" else tsdf.KERNEL_TMA) | (0 if stats else tsdf.NO_STATS)
    frames = room_seq(12, colour="on" if colour else "off", loop=1200)
    p = prm(24, 18, weight_sample=ws, batch_frames=4, flags=flags)
    compare(p, [frames])


# ---- colour and depth-only calls on one volume ----------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("ws", [1, 2])
@pytest.mark.parametrize("api", ["single", "batch", "device"])
def test_mixed_colour_and_depth_only_calls(built, api, ws):
    """colour, then depth-only, then colour: a stored colour survives the depth-only updates (in the constant-weight
    depth-only kernel too, which keeps the colour bytes while it counts weights in a register), and the next colour update
    averages against a weight that counts the depth-only frames"""
    frames = room_seq(12, loop=1200)
    calls = [frames[:4], [(d, None, T, K) for d, _, T, K in frames[4:8]], frames[8:]]
    gv = compare(prm(24, 18, weight_sample=ws, batch_frames=3), calls, api=api)
    assert gv["w"].max() >= 8


# ---- weight cap ------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("wmax", [1, 2, 3])
def test_saturated_weight_hot_path(built, wmax):
    """depth-only, constant sample weight, batches of 32: the hot kernel's unclamped counter runs far past weight_max"""
    frames = room_seq(70, colour="off", loop=4000)
    gv = compare(prm(24, 18, weight_max=wmax, batch_frames=32), [frames], max_ambiguous=0.1)
    assert gv["w"].max() == wmax


@pytest.mark.timeout(600)
def test_weight_reaches_255(built):
    """depth-only, constant sample weight: 264 frames of an almost still camera (8 full batches + 8), voxels reach the u8
    weight cap and stay there"""
    frames = room_seq(264, colour="off", loop=200000)
    # every frame flags a few voxels next to a pixel-rounding boundary, and the flags of 264 frames add up
    gv = compare(prm(24, 18, batch_frames=32), [frames], sample=400, max_ambiguous=0.2)
    assert gv["w"].max() == 255


# ---- bench shape -----------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_bench_shape_sampled(built):
    """640x480, 4 mm voxels, batches of 32, 64 frames (bench.py's instantiation); the float64 pass on ~2 000 blocks"""
    D, _, P, K = synth.make_frames(64, seed=0, loop_frames=1000)
    frames = [(D[i], None, P[i], K) for i in range(len(D))]
    # 640 px frames put each voxel near a pixel-rounding boundary of some frame more often than the small cases do
    compare(prm(640, 480, batch_frames=32, max_blocks=1 << 18, hash_slots=1 << 20), [frames], sample=2000, max_ambiguous=0.3)


# ---- pre-filtered depth ----------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("kernel", ["column", "tma"])
def test_filtered_depth(built, kernel):
    """k_alloc<1>: the bilateral filter's metres through the walk and the integrate kernels; the oracle and the float64
    fusion are fed the GPU-filtered images, which test_filter_gpu.py checks against the float64 filter"""
    frames = room_seq(10)
    flag = tsdf.KERNEL_COLUMN if kernel == "column" else tsdf.KERNEL_TMA
    p = prm(24, 18, batch_frames=4, flags=flag, depth_filter=1, depth_sigma_d=2.0, depth_sigma_r=0.05)
    metres = [tsdf.bilateral_filter(d, 1000.0, 2.0, 0.05) for d, _, _, _ in frames]
    compare(p, [frames], metres=metres)
