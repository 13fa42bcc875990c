"""The `.sens` scene driver scn_fuse_scene on its error paths, in both decode modes: the scene fails with the code and text of the
call that failed, prefixed by the .sens path, and a failed scene leaves no pooled volume behind."""
import zlib

import pytest

from scannet_b200 import ScnError, synth
from scannet_b200 import fuse as sfuse

pytestmark = pytest.mark.gpu
W, H = 160, 120
PARAMS = dict(voxel_size=0.008, trunc_base=0.04, max_blocks=50000, hash_slots=1 << 18)
ERR_FORMAT, ERR_CAPACITY = -4, -5


def _write_sens(path, n=12, corrupt=()):
    """zlib depth, no colour, every frame posed; frames in `corrupt` get a depth payload that does not inflate"""
    D, _, P, K = synth.make_frames(n, seed=31, width=W, height=H, loop_frames=400, with_color=False)
    with synth.SensWriter(str(path), n, (W, H), (0, 0), K, color_comp=0) as wr:
        for i in range(n):
            wr.add(b"", b"\x00garbage" * 9 if i in corrupt else zlib.compress(D[i].tobytes(), 6), P[i])
    return str(path)


@pytest.mark.parametrize("mode", ["gpu", "host"])
def test_full_voxel_heap_is_a_capacity_error(built, tmp_path, mode):
    sens = _write_sens(tmp_path / "scan.sens")
    with pytest.raises(ScnError) as e:
        sfuse.fuse_scene(sens, None, decode_mode=mode, **dict(PARAMS, max_blocks=64))
    assert e.value.code == ERR_CAPACITY and sens in str(e.value)


@pytest.mark.parametrize("mode", ["gpu", "host"])
def test_corrupt_depth_is_a_format_error_and_releases_the_pooled_volume(built, tmp_path, mode):
    clean, bad = _write_sens(tmp_path / "clean.sens"), _write_sens(tmp_path / "bad.sens", corrupt={5})
    before = sfuse.fuse_scene(clean, str(tmp_path / "before.ply"), decode_mode=mode, **PARAMS)
    with pytest.raises(ScnError) as e:
        sfuse.fuse_scene(bad, None, decode_mode=mode, **PARAMS)                  # same layout: takes the pooled volume
    assert e.value.code == ERR_FORMAT and bad in str(e.value)
    after = sfuse.fuse_scene(clean, str(tmp_path / "after.ply"), decode_mode=mode, **PARAMS)
    assert after["volume_reused"] == 0 and after["frames_integrated"] == before["frames_integrated"] == 12
    assert (tmp_path / "after.ply").read_bytes() == (tmp_path / "before.ply").read_bytes()
