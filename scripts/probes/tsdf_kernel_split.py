"""Where the fusion time goes on the GPU: k_alloc against the integrate kernel, per frame.

Renders bench.py's scene 0 (seeded box room, 1000 frames, 640x480) and fuses it one 32-frame batch at a time through
scn_tsdf_integrate_device, with a sync after every batch so that the allocation kernel of batch k+1 never overlaps the
integrate kernel of batch k (bench.py lets them overlap).  The two kernels' CUDA-event times (scn_tsdf_kernel_times) are
reported per frame, with the card's name and power limit read in the same run.  GPU only.
Usage: python scripts/probes/tsdf_kernel_split.py [--passes 5] [--batch 32]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import bench  # noqa: E402
from scannet_b200 import dist as sdist  # noqa: E402
from scannet_b200 import tsdf  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=5, help="timed passes over the scene (after one warm-up pass)")
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n = bench.SCENE_FRAMES
    sc, P = bench.scene_poses(n, sdist.scene_seed_for_rank(0) * 16, 1000)     # bench.py's scene 0 of rank 0
    d = bench.render_depth_torch(sc, P, dev)
    K = sc.intrinsics()
    torch.cuda.synchronize()
    fb = d[0].numel() * d.element_size()
    p = tsdf.default_params(batch_frames=args.batch, max_blocks=1 << 20, hash_slots=1 << 22)
    vol = tsdf.TsdfVolume(p, device=0)
    runs = []
    for it in range(args.passes + 1):
        vol.reset()
        vol.profile(True)
        for k0 in range(0, n, args.batch):
            m = min(args.batch, n - k0)
            vol.integrate_device(m, d.data_ptr() + k0 * fb, None, P[k0:k0 + m], K)
            vol.sync()
        a_ms, i_ms, nb, _ = vol.kernel_times()
        vol.profile(False)
        if it:                                                  # pass 0 warms up the modules and the volume
            runs.append({"alloc_us_per_frame": round(a_ms * 1e3 / n, 3), "integrate_us_per_frame": round(i_ms * 1e3 / n, 3),
                         "batches": nb})
    blocks = vol.stats().blocks_allocated
    vol.close()
    med = lambda key: float(np.median([r[key] for r in runs]))  # noqa: E731
    a, i = med("alloc_us_per_frame"), med("integrate_us_per_frame")
    out = {"card": card(), "frames": n, "batch": args.batch, "blocks": blocks, "runs": runs,
           "median": {"alloc_us_per_frame": a, "integrate_us_per_frame": i, "alloc_share": round(a / (a + i), 4)}}
    os.write(bench._REAL_STDOUT, (json.dumps(out) + "\n").encode())     # importing bench diverts fd 1 to stderr


if __name__ == "__main__":
    main()
