"""Where the time of one file -> TSDF scene goes (scn_fuse_scene reports) against the decode chunk size.
Usage: python scripts/probes/fuse_probe.py [frames] [color 0|1] [quick] > gpurun_out/fuse_probe.json   (the JSON goes to stdout)"""
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import bench  # noqa: E402
from scannet_b200 import fuse as sfuse  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
color = len(sys.argv) > 2 and sys.argv[2] == "1"
dev = torch.device("cuda:0")
out = {}
keys = ("wall_s", "total_s", "setup_s", "fuse_s", "buffers_s", "teardown_s", "decode_wait_s", "integrate_s", "depth_decode_s", "depth_pack_s", "depth_kernel_s",
        "color_decode_s", "color_host_s", "color_entropy_s", "color_convert_s", "frames_per_s_incl_decode")
with tempfile.TemporaryDirectory() as d:
    p = os.path.join(d, "scene.sens")
    bench.make_sens_file(p, n, 100, dev, with_color=color)
    over = dict(max_blocks=1 << 22, hash_slots=1 << 24) if color else {}
    sweep = ("1024", "512", "2048") if len(sys.argv) <= 3 else ("1024",)
    for chunk in sweep:
        os.environ["SCN_FUSE_CHUNK"] = chunk
        runs = []
        for rep_i in range(2 if len(sys.argv) <= 3 else 4):
            t0 = time.perf_counter()
            rep = sfuse.fuse_scene(p, None, decode_mode="gpu", device=0, **over)
            rep["wall_s"] = time.perf_counter() - t0
            runs.append({k: round(rep[k], 4) for k in keys})
        out[f"chunk_{chunk}"] = runs
os.write(bench._REAL_STDOUT, (json.dumps(out, indent=1) + "\n").encode())
