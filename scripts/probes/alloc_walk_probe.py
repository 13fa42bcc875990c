"""What k_alloc's walk really executes, per warp and per lane, and where a CTA's time goes.

Builds two private copies of the library in a temporary directory: csrc/tsdf.cu compiled with -DSCN_ALLOC_PROBE=1 (counters)
and =2 (clock64 per phase), hooks in scripts/probes/alloc_walk_probe.cuh, linked with the other objects of `make lib`
(build/obj).  Each copy fuses bench.py's scene 0 (seeded box room, 1000 frames, 640x480, batches of 32) once and the
counters are read back.  "Warp" = the lanes that execute a step together.  The clock shares are of lane 0 of every warp,
summed over the CTA's 8 warps; a frame whose lane 0 has no valid depth counts its set-up as walk.  GPU only.
Usage: python scripts/probes/alloc_walk_probe.py [--batch 32]"""
import argparse
import ctypes as C
import glob
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

NAMES = ["warp_steps", "warp_steps_miss", "lane_steps", "lane_miss", "miss_flag", "miss_claim", "miss_global", "collide",
         "flag_lanes", "flag_addrs", "warp_frames", "warp_max_steps", "lane_frames", "keys", "touch", "ctas", "head0", "head1", "head2", "head3",
         "clk_prologue", "clk_setup", "clk_walk", "clk_barrier", "clk_flush"]          # AllocProbeCounter, in order


def build(mode, out):
    """the library with tsdf.cu compiled as probe `mode`; the compiler and flags are the Makefile's"""
    objs = [o for o in sorted(glob.glob(os.path.join(ROOT, "build", "obj", "*.o"))) if os.path.basename(o) != "tsdf.o"]
    if not objs:
        sys.exit("build/obj is empty: run `make lib` first")
    mk = subprocess.run(["make", "-s", "-C", ROOT, "--eval=probe-flags: ; @echo $(NVCC) $(NVFLAGS)", "probe-flags"],
                        capture_output=True, text=True, check=True).stdout.split()
    obj, so = os.path.join(out, f"tsdf_probe{mode}.o"), os.path.join(out, f"libscannet_b200_probe{mode}.so")
    subprocess.run(mk + [f"-DSCN_ALLOC_PROBE={mode}", "-I", HERE, "-c", os.path.join(ROOT, "scannet_b200", "csrc", "tsdf.cu"), "-o", obj],
                   check=True, cwd=ROOT, capture_output=True)
    subprocess.run([mk[0], "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", so, obj] + objs +
                   ["-ccbin", "/usr/bin/g++", "-cudart", "static", "-lpthread"], check=True, capture_output=True)
    return so


def run(so, d, P, K, n, batch):
    """one pass of the scene through the library at `so`; returns the counters"""
    from scannet_b200 import _lib, tsdf
    _lib.LIB_PATH, _lib._lib = so, None
    p = tsdf.default_params(batch_frames=batch, max_blocks=1 << 20, hash_slots=1 << 22)
    vol = tsdf.TsdfVolume(p, device=0)
    fb = d[0].numel() * d.element_size()
    out = (C.c_uint64 * len(NAMES))()
    assert _lib.lib().scn_alloc_probe_read(out, len(NAMES)) == len(NAMES)            # zero them
    for k0 in range(0, n, batch):
        m = min(batch, n - k0)
        vol.integrate_device(m, d.data_ptr() + k0 * fb, None, P[k0:k0 + m], K)
    vol.sync()
    assert _lib.lib().scn_alloc_probe_read(out, len(NAMES)) == len(NAMES)
    vol.close()
    return dict(zip(NAMES, [int(v) for v in out]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    import torch
    import bench
    from scannet_b200 import dist as sdist
    with tempfile.TemporaryDirectory() as tmp:
        libs = [build(1, tmp), build(2, tmp)]
        dev = torch.device("cuda:0")
        n = bench.SCENE_FRAMES
        sc, P = bench.scene_poses(n, sdist.scene_seed_for_rank(0) * 16, 1000)     # bench.py's scene 0 of rank 0
        d = bench.render_depth_torch(sc, P, dev)
        torch.cuda.synchronize()
        c, t = (run(so, d, P, sc.intrinsics(), n, args.batch) for so in libs)
    clk = {k: t[k] for k in NAMES if k.startswith("clk_")}
    tot = float(sum(clk.values())) or 1.0
    r = lambda a, b: round(a / b, 3) if b else 0.0  # noqa: E731
    out = {
        "card": torch.cuda.get_device_name(0), "frames": n, "batch": args.batch,
        "per_frame": {
            "warp_steps": r(c["warp_steps"], n), "warp_steps_with_a_miss": r(c["warp_steps_miss"], n),
            "lane_steps": r(c["lane_steps"], n), "lane_misses": r(c["lane_miss"], n),
            "miss_key_present_flag_clear": r(c["miss_flag"], n), "miss_claim": r(c["miss_claim"], n),
            "miss_global_fallback": r(c["miss_global"], n), "collision_probes": r(c["collide"], n),
            "touch_block_calls": r(c["touch"], n)},
        "warp_miss_share": r(c["warp_steps_miss"], c["warp_steps"]),
        "lane_miss_share": r(c["lane_miss"], c["lane_steps"]),
        "lanes_per_warp_step": r(c["lane_steps"], c["warp_steps"]),
        "lanes_per_flag_address": r(c["flag_lanes"], c["flag_addrs"]),
        "steps_per_lane_mean": r(c["lane_steps"], c["lane_frames"]),
        "steps_per_lane_warp_max_mean": r(c["warp_max_steps"], c["warp_frames"]),
        "distinct_keys_per_cta": r(c["keys"], c["ctas"]),
        "lane_groups_per_warp_at_frame_head": [r(c[f"head{j}"], 8 * c["ctas"]) for j in range(4)],   # (the last batch's groups are full too: 1000 = 31 * 32 + 8)
        "clock_share": {k[4:]: round(v / tot, 4) for k, v in clk.items()},
        "clock_ticks_per_cta_warp": r(tot, 8 * t["ctas"]),
        "raw": {"counters": c, "clocks": t}}
    os.write(bench._REAL_STDOUT, (json.dumps(out) + "\n").encode())     # importing bench diverts fd 1 to stderr


if __name__ == "__main__":
    main()
