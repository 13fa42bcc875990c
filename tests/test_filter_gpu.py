"""Depth bilateral pre-filter (§8(f)2).  The in-tree reference is itself a CUDA kernel
(AnnotationTools/Filter2dAnnotations/filter.cu:210-247) using exp/expf, which are not correctly rounded and differ
between CUDA and libm: the CUDA kernel is compared with the CPU restatement to a TOLERANCE of 2e-6 relative
(≈ a dozen float ulps; observed error is far smaller), invalid (-inf) pixels must coincide exactly.  The fused path
(params.depth_filter) is then checked bit-exactly against the oracle fed with the GPU-filtered image."""
import numpy as np
import pytest

import oracle_bindings as ob
from scannet_b200 import synth, tsdf

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("sd,sr,wh", [(2.0, 0.05, (160, 120)), (2.0, 0.1, (97, 61)), (1.0, 0.02, (64, 48)), (3.5, 0.05, (80, 60))])
def test_filter_matches_cpu_restatement(built, sd, sr, wh):
    D, _, _, _ = synth.make_frames(1, seed=5, width=wh[0], height=wh[1], noise_mm=4.0, drop=0.08, with_color=False)
    g = tsdf.bilateral_filter(D[0], 1000.0, sd, sr)
    o = ob.oracle_bilateral(D[0], 1000.0, sd, sr)
    inv = np.isinf(o)
    assert (np.isinf(g) == inv).all() and (g[inv] == -np.inf).all() and (D[0] == 0)[inv].all()
    rel = np.abs(g[~inv] - o[~inv]) / np.abs(o[~inv])
    assert rel.max() < 2e-6, rel.max()
    # it is a smoothing filter: noise goes down, edges stay
    raw = D[0].astype(np.float32) / 1000.0
    assert np.abs(g[~inv] - raw[~inv]).max() < 0.2


@pytest.mark.parametrize("sd,sr,wh", [(2.0, 0.05, (160, 120)), (2.0, 0.1, (97, 61)), (1.0, 0.02, (64, 48)), (3.5, 0.05, (80, 60)),
                                      (4.0, 0.05, (80, 60)), (0.1, 0.05, (80, 60))])
def test_filter_matches_float64(built, sd, sr, wh):
    """Against the float64 statement of the filter (tests/tsdf_reference.py:bilateral_f64), which shares no arithmetic with
    the kernel or the oracle.  Bound from the number of taps n = (2r + 1)^2: binary32 sums of n weights and n weighted depths
    (n roundings each) and weights within ~4 ulp (expf, the double exp rounded to float, the product) put the weighted
    mean within (2n + 8) ulp of the largest depth of the window."""
    import tsdf_reference as tref
    D, _, _, _ = synth.make_frames(1, seed=5, width=wh[0], height=wh[1], noise_mm=4.0, drop=0.08, with_color=False)
    g = tsdf.bilateral_filter(D[0], 1000.0, sd, sr)
    ref, taps = tref.bilateral_f64(D[0], 1000.0, sd, sr)
    inv = np.isinf(ref)
    assert (np.isinf(g) == inv).all() and (g[inv] == -np.inf).all()
    err = np.abs(g[~inv].astype(np.float64) - ref[~inv])
    assert err.max() <= (2 * taps + 8) * 2.0 ** -24 * np.abs(ref[~inv]).max(), err.max()
    assert (err > 0).any()                                     # the comparison is not with itself


def test_fused_filter_path_bit_exact_given_filtered_depth(built):
    p = tsdf.default_params(width=128, height=96, max_blocks=1 << 15, hash_slots=1 << 17, batch_frames=3,
                            depth_filter=1, depth_sigma_d=2.0, depth_sigma_r=0.05)
    D, C, P, K = synth.make_frames(5, seed=9, width=128, height=96, loop_frames=200, noise_mm=3.0, drop=0.03, invalid_pose_every=4)
    vol = tsdf.TsdfVolume(p, device=0)
    vol.integrate_batch(D, C, P, K); vol.sync()
    gx, gv = vol.download_blocks(); st = vol.stats(); vol.close()
    o = ob.OracleTsdf(p, threads=4)
    for i in range(len(D)):
        o.integrate_metres(tsdf.bilateral_filter(D[i], 1000.0, 2.0, 0.05), C[i], P[i], K)
    ox, ov = o.export()
    assert gx.shape == ox.shape and (gx == ox).all() and gv.tobytes() == ov.tobytes()
    assert st.voxels_updated == o.counters()["total_updated"] and st.frames_skipped == 1
    # and filtering changed something compared with the unfiltered volume
    p2 = tsdf.default_params(width=128, height=96, max_blocks=1 << 15, hash_slots=1 << 17, batch_frames=3)
    v2 = tsdf.TsdfVolume(p2, device=0); v2.integrate_batch(D, C, P, K); v2.sync()
    _, uv = v2.download_blocks(); v2.close()
    assert uv.tobytes() != gv.tobytes()


def test_params_file_enables_filter(built, tmp_path):
    f = tmp_path / "p.txt"
    f.write_text("s_depthSigmaD = 2.0f;\ns_depthSigmaR = 0.05f;\t//x\ns_depthFilter = true;\n")
    p = tsdf.params_from_file(str(f))
    assert p.depth_filter == 1 and abs(p.depth_sigma_r - 0.05) < 1e-9 and p.depth_sigma_d == 2.0
