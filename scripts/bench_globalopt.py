"""Measures the global optimiser (csrc/globalopt.cu, DESIGN.md §6k) alone: keyframes, edges, pairs per Gauss-Newton iteration and
the GPU phase times, on the drifted 300-frame orbit (30 keyframes) and at the configs[2] stand-in scale (5,578 frames -> 558
keyframes); the smaller case is also compared with the oracle bit for bit.  Then `recons --global` end to end against plain `recons`
on the same 300-frame .sens.  Prints one JSON line per case, with the card's name and power limit read in the same run.

    python scripts/bench_globalopt.py [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import globalopt_bindings as gb  # noqa: E402
import recons_bindings as rb  # noqa: E402
from scannet_b200 import recons, tsdf  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def case(n_frames, check_oracle, W=320, H=240):
    sc = gb.scene(W, H)
    gp = recons.global_default_params()
    n = n_frames // gp.submap_size
    D, P, Q = gb.loop_keyframes(sc, n)
    vol = tsdf.TsdfVolume(tsdf.default_params(width=W, height=H, max_blocks=1 << 10, hash_slots=1 << 12, batch_frames=1))
    opt = recons.GlobalOptimizer(vol, gp)
    opt.add_keyframes(D, Q, sc.intrinsics())
    t = time.perf_counter()
    poses, rep = opt.solve()
    wall = time.perf_counter() - t
    out = dict(frames=n_frames, depth=f"{W}x{H}", keyframe_size=f"{gp.width}x{gp.height}", solve_wall_s=wall,
               ate_before_mm=gb.ate(Q, P)[0] * 1000, ate_after_mm=gb.ate(poses, P)[0] * 1000,
               **{k: v for k, v in rep.items() if k != "rss_iter"})
    out["pairs_per_iteration"] = rep["pairs_before"]
    if check_oracle:
        o = gb.OracleGlobal(gp, W, H)
        for k in range(n):
            o.add_keyframe(rb.metres(D[k]), sc.intrinsics(), Q[k])
        want, orep = o.solve()
        out["oracle_bit_identical"] = bool(want.tobytes() == poses.tobytes() and all(orep[k] == rep[k] for k in gb.COUNTERS))
    return out


def end_to_end(n_frames=300, W=320, H=240):
    """plain `recons` against `recons --global` on the same .sens (converter-style poses), host clock around each call"""
    import shutil
    import tempfile
    from test_recons_gpu import PARAMS, frames, scene
    sc = scene(W, H, 2)
    D, C_, P = frames(sc, n_frames, 1.0, 0.02)
    conv = P.copy(); conv[1:] = np.eye(4, dtype=np.float32)
    p = tsdf.default_params(voxel_size=0.01, trunc_base=0.06, trunc_scale=0.02)
    tp, gp = recons.default_params(), recons.global_default_params()
    for f in PARAMS:
        tsdf.params_from_file(f, p); recons.params_from_file(f, tp); recons.global_params_from_file(f, gp)
    out = dict(frames=n_frames, depth=f"{W}x{H}")
    with tempfile.TemporaryDirectory() as d:
        from scannet_b200 import synth
        src = os.path.join(d, "s.sens")
        synth.write_sens(src, D, C_, conv, sc.intrinsics(), depth_comp=1, color_comp=0)
        for k in ("plain", "global", "plain", "global"):                 # the first pair warms up, the second is reported
            shutil.copyfile(src, os.path.join(d, k + ".sens"))
            t = time.perf_counter()
            if k == "plain":
                rep = recons.recons_scene(os.path.join(d, k + ".sens"), os.path.join(d, k + ".ply"), None, p, tp)
            else:
                rep, grep = recons.recons_scene_global(os.path.join(d, k + ".sens"), os.path.join(d, k + ".ply"), None, p, tp, gp)
            out[k + "_s"] = time.perf_counter() - t
        for k in ("plain", "global"):
            from test_recons_gpu import masked
            out[k + "_ate_mm"] = rb.pose_errors(masked(os.path.join(d, k + ".sens"))[1], P)[0] * 1000
        out.update({"global_" + k: v for k, v in grep.items() if k != "rss_iter"})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = [dict(card=card())]
    for n_frames, chk in ((300, True), (5578, False)):
        res.append(case(n_frames, chk))
        print(json.dumps(res[-1]), flush=True)
    res.append(end_to_end())
    print(json.dumps(res[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res[0]))


if __name__ == "__main__":
    main()
