"""k_alloc's shared-memory cell map under load, bit for bit against oracle/tsdf_oracle.c.

The map keeps one flag byte per frame of a CTA's group of 4 frames.  These cases put several frames through the paths
around it: 16x16-pixel regions that see far more distinct blocks than the map has room for near a cell's home slot (1 mm
voxels and noisy depth: every ray holds its own cells, so cells find 8 occupied slots in a row and go to the global table
with their frame's bit), for batches that make groups of 1, 3 and 4 frames and a group after a full one; and the
pre-filtered-depth variant of the kernel through a full group of 4 frames."""
import numpy as np
import pytest

import oracle_bindings as ob
from scannet_b200 import synth, tsdf

pytestmark = pytest.mark.gpu


def compare(p, D, P, K, integrate):
    vol = tsdf.TsdfVolume(p, device=0)
    try:
        vol.integrate_batch(D, None, P, K)
        vol.sync()
        gx, gv = vol.download_blocks()
        st = vol.stats()
    finally:
        vol.close()
    o = ob.OracleTsdf(p, threads=8)
    for i in range(len(D)):
        integrate(o, i)
    ox, ov = o.export()
    oc = o.counters()
    o.close()
    assert gx.shape == ox.shape and (gx == ox).all(), f"block sets differ ({len(gx)} vs {len(ox)})"
    assert gv.tobytes() == ov.tobytes(), "voxels differ"
    assert st.voxels_updated == oc["total_updated"] and st.blocks_visited == oc["total_touched"]
    assert st.frames_integrated == oc["frames_done"]
    return len(ox)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("batch", [1, 3, 4, 5, 32])
def test_crowded_map_with_several_frames_in_a_group(built, batch):
    W, H, n = 64, 48, 6
    D, _, P, K = synth.make_frames(n, seed=23, width=W, height=H, loop_frames=300, noise_mm=12.0, with_color=False)
    p = tsdf.default_params(width=W, height=H, voxel_size=0.001, max_blocks=1 << 19, hash_slots=1 << 21, batch_frames=batch)
    blocks = compare(p, D, P, K, lambda o, i: o.integrate(D[i], None, P[i], K))
    # 12 regions of 16x16 pixels: each sees more than twice as many distinct blocks per frame as its map has slots
    assert blocks > 12 * n * 2 * 1024, blocks


def test_filtered_depth_variant_through_a_full_group(built):
    W, H, n = 128, 96, 9                                         # batches of 8 + 1: groups of 4, 4 and 1 frames
    D, _, P, K = synth.make_frames(n, seed=9, width=W, height=H, loop_frames=200, noise_mm=3.0, drop=0.03, with_color=False)
    p = tsdf.default_params(width=W, height=H, max_blocks=1 << 15, hash_slots=1 << 17, batch_frames=8,
                            depth_filter=1, depth_sigma_d=2.0, depth_sigma_r=0.05)
    compare(p, D, P, K, lambda o, i: o.integrate_metres(tsdf.bilateral_filter(D[i], 1000.0, 2.0, 0.05), None, P[i], K))
