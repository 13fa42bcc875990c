#!/usr/bin/env python
"""Freezes the TSDF spec: hashes of the CPU oracle's output on seeded inputs -> tests/golden/tsdf_spec_golden.json.
The reference has no TSDF source, so this does not pin the oracle to the reference — it pins the oracle (and with it
the CUDA path, which must match it bit for bit) against accidental drift of this repo's own spec (DESIGN.md §3)."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_bindings as ob  # noqa: E402
from scannet_b200 import synth  # noqa: E402
from scannet_b200._lib import TsdfParams  # noqa: E402


def params(w, h, **kw):
    p = TsdfParams(); p.voxel_size = 0.004; p.trunc_base = 0.02; p.trunc_scale = 0.01; p.depth_min = 0.1; p.depth_max = 6.0
    p.max_integration_distance = 4.0; p.weight_sample = 1; p.weight_max = 255; p.width = w; p.height = h; p.depth_shift = 1000.0
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def run(case):
    w, h = case["wh"]
    D, C, P, K = synth.make_frames(case["frames"], seed=case["seed"], width=w, height=h, loop_frames=case["loop"],
                                   noise_mm=case["noise"], drop=case["drop"], invalid_pose_every=case["inv"])
    o = ob.OracleTsdf(params(w, h, **case["over"]), threads=4)
    for i in range(len(D)):
        o.integrate(D[i], C[i] if case["color"] else None, P[i], K)
    xyz, vox = o.export()
    mx, mc, mt = o.extract_mesh()
    c = o.counters()
    return {"blocks": int(len(xyz)), "updated": c["total_updated"], "touched": c["total_touched"], "skipped": c["frames_skipped"],
            "volume_sha256": hashlib.sha256(xyz.tobytes() + vox.tobytes()).hexdigest(),
            "mesh_sha256": hashlib.sha256(mx.tobytes() + mc.tobytes() + mt.tobytes()).hexdigest(),
            "mesh_verts": int(len(mx)), "mesh_faces": int(len(mt))}


CASES = [
    {"name": "color_noise", "wh": [96, 72], "frames": 5, "seed": 21, "loop": 200, "noise": 1.5, "drop": 0.02, "inv": 0, "color": True, "over": {}},
    {"name": "depth_only_invalid_pose", "wh": [128, 96], "frames": 6, "seed": 22, "loop": 90, "noise": 0.0, "drop": 0.1, "inv": 4, "color": False, "over": {}},
    {"name": "weighted", "wh": [80, 60], "frames": 9, "seed": 23, "loop": 3000, "noise": 0.5, "drop": 0.0, "inv": 0, "color": True,
     "over": {"weight_sample": 10, "weight_max": 30}},
    # per-sample weight past the 512-entry reciprocal table of the integrate kernel (w1 up to 1500)
    {"name": "heavy_weight_sample", "wh": [64, 48], "frames": 4, "seed": 24, "loop": 300, "noise": 0.5, "drop": 0.01, "inv": 0, "color": True,
     "over": {"weight_sample": 1000}},
    {"name": "voxel_1mm", "wh": [24, 18], "frames": 3, "seed": 25, "loop": 300, "noise": 0.0, "drop": 0.0, "inv": 0, "color": True,
     "over": {"voxel_size": 0.001}},
    {"name": "voxel_2cm_no_trunc_scale", "wh": [72, 54], "frames": 5, "seed": 26, "loop": 100, "noise": 1.0, "drop": 0.02, "inv": 3, "color": False,
     "over": {"voxel_size": 0.02, "trunc_scale": 0.0}},
]

if __name__ == "__main__":
    out = {"spec": "TSDF spec v1.1 + marching cubes (DESIGN.md §3, §6)", "cases": []}
    for c in CASES:
        r = run(c); out["cases"].append({**c, **r}); print(c["name"], r)
    L = ob.tsdf_oracle_lib(); n = np.zeros(256, np.uint8); t = np.zeros((256, 36), np.uint8)
    L.oracle_mc_table(n.ctypes.data, t.ctypes.data)
    out["mc_table_sha256"] = hashlib.sha256(n.tobytes() + t.tobytes()).hexdigest()
    with open(os.path.join(ROOT, "tests", "golden", "tsdf_spec_golden.json"), "w") as fh:
        json.dump(out, fh, indent=1)
