#!/usr/bin/env python
"""Free-space benchmark (DESIGN.md §6h): the `freespace` stage (scn_freespace_scene, .sens -> .grid at 5 cm) on the BASELINE.json
configs[2] stand-in — the 5,578-frame synthetic scan bench.py's `pipeline_c3` builds (bench.make_sens_file; 640x480 zlib depth).
Reports the envelope and output boxes, the label counts, frames/s including decode, the decode / classify / crop times, the
(brick, frame) pairs classified and culled (best of 3 runs after a warm-up), the card and its power limit, then the oracle on
all host threads over a bounded sample of frames (labelled as sampled) and whether the GPU and the oracle agree bit for bit on
that sample.  Everything is written to a temporary directory; prints one JSON object.
Usage: python scripts/bench_freespace.py [n_frames] [oracle_sample_frames]"""
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 5578
    n_sample = int(sys.argv[2]) if len(sys.argv) > 2 else 64
    import torch
    import bench                                                # the stand-in scan generator; bench diverts stdout to stderr
    import freespace_bindings as fb
    from scannet_b200 import freespace, sens
    out = {"frames": n, "card": card()}
    p = freespace.default_params()
    out["params"] = {k: getattr(p, k) for k, _ in freespace.FreespaceParams._fields_}
    with tempfile.TemporaryDirectory() as d:
        path, grid = os.path.join(d, "scene.sens"), os.path.join(d, "scene.grid")
        _, out["generate_s"] = bench.make_sens_file(path, n, 7, torch.device("cuda:0"), with_color=False)
        freespace.freespace_scene(path, grid, p)                                                   # warm-up
        reps = [freespace.freespace_scene(path, grid, p) for _ in range(3)]
        rep = min(reps, key=lambda r: r["total_s"])
        out.update({k: rep[k] for k in ("frames_used", "frames_skipped_pose", "envelope_lo", "envelope_dims", "output_lo", "output_dims",
                                        "voxels_free", "voxels_occupied", "voxels_unknown", "pairs_classified", "pairs_culled")})
        out["envelope_voxels"] = int(np.prod(rep["envelope_dims"]))
        out["frames_per_s_incl_decode"] = round(rep["frames_used"] / rep["total_s"], 1)
        out["ms"] = {"decode": round(rep["decode_s"] * 1e3, 2), "classify": round(rep["classify_ms"], 2), "crop_download": round(rep["crop_ms"], 2),
                     "write": round(rep["write_s"] * 1e3, 2), "total": round(rep["total_s"] * 1e3, 2)}
        out["total_ms_runs"] = [round(r["total_s"] * 1e3, 2) for r in reps]
        out["pairs_classified_fraction"] = round(rep["pairs_classified"] / max(1, rep["pairs_classified"] + rep["pairs_culled"]), 5)
        # the oracle on a bounded sample: every (n // n_sample)-th frame, over the same envelope, against the handle on the same frames
        sf = sens.SensFile(path)
        idx = list(range(0, n, max(1, n // n_sample)))[:n_sample]
        info = sf.info
        W, H = info.depth_width, info.depth_height
        K = np.asarray(info.depth_intrinsic, np.float32).reshape(4, 4)
        D = np.stack([sf.depth(i) for i in idx]); P = np.stack([sf.pose(i) for i in idx])
    lo, dims = rep["envelope_lo"], rep["envelope_dims"]                                       # the whole scan's envelope
    with freespace.FreeSpace(lo, dims, W, H, params=p) as h:
        h.integrate(D, P, K)
        g = h.download()
    threads = os.cpu_count() or 1
    t0 = time.perf_counter()
    o = fb.OracleCounts(p, lo, dims, W, H, threads=threads).integrate(D, P, K).result()
    oracle_s = time.perf_counter() - t0
    out["oracle_sampled"] = {"frames": len(idx), "threads": threads, "envelope_dims": list(dims), "seconds": round(oracle_s, 3),
                             "frames_per_s": round(len(idx) / oracle_s, 2)}
    out["bit_identical_to_oracle_on_sample"] = bool(tuple(g[0]) == tuple(o[0]) and g[1] == o[1] and all(a.tobytes() == b.tobytes()
                                                                                                          for a, b in zip(g[2:], o[2:])))
    bench.emit(out)


if __name__ == "__main__":
    main()
