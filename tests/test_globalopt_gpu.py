"""GPU global optimiser (csrc/globalopt.cu) against the CPU oracle (oracle/globalopt_oracle.c), bit for bit: edge list, pairs per
edge, sum of r^2 per Gauss-Newton iteration, final pose bytes and report counters; and the optimiser's refusals."""
import numpy as np
import pytest

import globalopt_bindings as gb
import recons_bindings as rb
from scannet_b200 import ScnError, recons, tsdf

pytestmark = pytest.mark.gpu

CASES = [  # depth size, keyframe size, filter, keyframes, zero-depth keyframe, keyframe from another scene, least ATE reduction
    ((320, 240), (80, 60), 1, 12, 7, 3, 5.0),
    ((640, 480), (80, 60), 0, 10, None, None, 5.0),
    ((160, 120), (40, 30), 0, 12, 4, 9, 1.5),       # 40 x 30 keyframes and two of twelve cut loose: measured 4.5 -> 2.2 cm in the oracle
]


def volume_params(W, H, depth_filter):
    return tsdf.default_params(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02, width=W, height=H, max_blocks=1 << 10,
                               hash_slots=1 << 12, batch_frames=1, depth_filter=depth_filter, depth_sigma_d=2.0, depth_sigma_r=0.05)


@pytest.mark.parametrize("case", CASES, ids=["320to80-filter", "640to80", "160to40-raw"])
def test_optimiser_bit_identical_to_oracle(built, case):
    (W, H), (kw, kh), filt, n, zero_at, bad, gain = case
    sc = gb.scene(W, H)
    D, P, Q = gb.loop_keyframes(sc, n, bad=bad)
    if zero_at is not None:
        D[zero_at] = 0
    K = sc.intrinsics()
    gp = recons.global_default_params(width=kw, height=kh)
    vol = tsdf.TsdfVolume(volume_params(W, H, filt))
    opt = recons.GlobalOptimizer(vol, gp)
    opt.add_keyframes(D[:n // 2], Q[:n // 2], K)          # two calls: the keyframes accumulate
    opt.add_keyframes(D[n // 2:], Q[n // 2:], K)
    got, rep = opt.solve()
    ora = gb.OracleGlobal(gp, W, H)
    for k in range(n):
        m = tsdf.bilateral_filter(D[k], 1000.0, 2.0, 0.05) if filt else rb.metres(D[k])
        ora.add_keyframe(m, K, Q[k])
    want, orep = ora.solve()
    ge, oe = opt.edges(), ora.edges()
    assert [(e["i"], e["j"], e["loop"], e["removed"]) for e in ge] == [(e["i"], e["j"], e["loop"], e["removed"]) for e in oe]
    for g, o in zip(ge, oe):
        if not o["removed"]:
            assert g["pairs"] == o["pairs"] and np.float64(g["rss"]).tobytes() == np.float64(o["rss"]).tobytes(), (g, o)
    for k in gb.COUNTERS:
        assert np.asarray(rep[k]).tobytes() == np.asarray(orep[k]).tobytes(), (k, rep[k], orep[k])
    assert np.asarray(rep["rss_iter"]).tobytes() == np.asarray(orep["rss_iter"]).tobytes()
    assert got.tobytes() == want.tobytes()
    assert rep["keyframes"] == n and not rep["rejected"] and rep["edges_loop"] > 0
    for k in (zero_at, bad):
        if k is not None:
            assert got[k].tobytes() == Q[k].tobytes()
            assert all(e["removed"] for e in ge if k in (e["i"], e["j"]))
    keep = [k for k in range(n) if k not in (zero_at, bad)]
    before, after = gb.ate(Q[keep], P[keep]), gb.ate(got[keep], P[keep])
    print(f"{W}x{H}->{kw}x{kh}: {rep['edges_consecutive']}+{rep['edges_loop']} edges, {rep['edges_removed']} removed, ATE "
          f"{before[0] * 1000:.1f} -> {after[0] * 1000:.2f} mm; GPU ms maps {rep['keyframe_maps_ms']:.2f} overlap {rep['overlap_ms']:.2f} "
          f"linearise {rep['linearise_ms']:.2f} pcg {rep['pcg_ms']:.2f} verify {rep['verify_ms']:.2f}")
    assert after[0] <= before[0] / gain
    assert min(rep[k] for k in ("overlap_ms", "linearise_ms", "pcg_ms", "verify_ms", "keyframe_maps_ms")) > 0


def test_too_many_keyframes_is_a_capacity_error(built):
    sc = gb.scene(160, 120)
    D, P, Q = gb.loop_keyframes(sc, 4)
    vol = tsdf.TsdfVolume(volume_params(160, 120, 0))
    opt = recons.GlobalOptimizer(vol, recons.global_default_params(width=40, height=30, max_keyframes=3))
    opt.add_keyframes(D[:2], Q[:2], sc.intrinsics())
    with pytest.raises(ScnError) as e:
        opt.add_keyframes(D[2:], Q[2:], sc.intrinsics())
    assert e.value.code == -5
    poses, rep = opt.solve()                                 # nothing of the refused call was added
    assert rep["keyframes"] == 2 and poses.shape == (2, 4, 4)


def test_resolution_not_a_power_of_two_divisor_is_refused(built):
    vol = tsdf.TsdfVolume(volume_params(160, 120, 0))
    with pytest.raises(ScnError):
        recons.GlobalOptimizer(vol, recons.global_default_params(width=60, height=45))
