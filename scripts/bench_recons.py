"""Tracker benchmark (DESIGN.md §6j): a 300-frame loop around a synthetic room (640x480 depth, 1 mm noise, 2 % dropouts, 1 cm
voxels, tracking at 320x240), tracked and integrated on the GPU from device-resident frames.  Prints frames/s, kernel launches per
frame, the trajectory error against the generator's poses, the oracle on the first 64 frames (bit-identical or not), and the card's
name and power limit read in the same run; then the same frames as a .sens through scn_recons_scene (decode, tracking, marching
cubes, PLY and .sens write), with the phase split from CUDA events."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import recons_bindings as rb  # noqa: E402
from scannet_b200 import recons, synth, tsdf  # noqa: E402


def main():
    n, W, H = 300, 640, 480
    sc = synth.BoxRoomScene(size=(5.0, 4.0, 3.0), n_spheres=10, seed=2, width=W, height=H, fx=synth.FX, fy=synth.FY, cx=(W - 1) / 2, cy=(H - 1) / 2)
    K = sc.intrinsics()
    P = np.stack([sc.orbit_pose(i, 300, height=2.2) for i in range(n)])
    R = [sc.render(P[i], noise_mm=1.0, drop=0.02, frame_seed=i) for i in range(n)]
    D = np.stack([r[0] for r in R]); C = np.stack([r[1] for r in R])
    vp = tsdf.default_params(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02, max_integration_distance=4.0, width=W, height=H,
                             max_blocks=1 << 17, hash_slots=1 << 19, batch_frames=1, depth_filter=1, depth_sigma_d=2.0, depth_sigma_r=0.05)
    tp = recons.default_params()
    dd = torch.from_numpy(D.view(np.int16)).to("cuda:0"); dc = torch.from_numpy(C).to("cuda:0")
    runs = []
    for rep in range(3):                            # the first run is warm-up
        vol = tsdf.TsdfVolume(vp); tr = recons.Tracker(vol, tp)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        got = tr.frames_device(n, dd.data_ptr(), dc.data_ptr(), K, P[0])
        torch.cuda.synchronize(); dt = time.perf_counter() - t0
        runs.append((dt, tr.stats(), got, vol))
    dt, st, got, vol = runs[-1]
    te, re = rb.pose_errors([g["cam2world"] for g in got], P)
    ora = rb.OracleTracker(vp, tp)
    same = True
    for i in range(64):
        o = ora.frame(tsdf.bilateral_filter(D[i], 1000.0, 2.0, 0.05), C[i], K, P[0])
        same &= o["cam2world"].tobytes() == got[i]["cam2world"].tobytes() and o["pairs"] == got[i]["pairs"]
    # the scene driver on the same frames from a .sens (zlib depth, raw colour, identity poses after frame 0): decode included
    conv = P.copy(); conv[1:] = np.eye(4, dtype=np.float32)
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "loop.sens")
        synth.write_sens(path, D, C, conv, K, depth_comp=1, color_comp=0)
        vp.batch_frames = 32
        reps = [recons.recons_scene(path, os.path.join(td, "loop.ply"), os.path.join(td, "out.sens"), vp, tp) for _ in range(2)]
    rep = reps[-1]
    scene = {k: round(rep[k], 4) if isinstance(rep[k], float) else rep[k] for k in (
        "frames", "frames_lost", "recons_s", "decode_s", "track_s", "filter_pyramid_ms", "icp_ms", "integrate_ms", "raycast_ms", "mc_s", "ply_s",
        "sens_s", "total_s", "kernel_launches")}
    scene["frames_per_s_incl_decode"] = round(rep["frames"] / rep["recons_s"], 1)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"frames": n, "seconds": [round(r[0], 4) for r in runs], "frames_per_s": round(n / dt, 1),
                      "launches_per_frame": round(st["kernel_launches"] / n, 2), "lost": int(sum(g["lost"] for g in got)),
                      "ate_m": round(te, 5), "max_rot_deg": round(re, 4), "oracle_first_64_bit_identical": bool(same), "scene_driver": scene, "gpu": smi}))


if __name__ == "__main__":
    main()
