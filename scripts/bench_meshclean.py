#!/usr/bin/env python
"""Mesh-cleaning benchmark (DESIGN.md §6f): clean.mlx (merge 0.0010689 m, duplicate faces, pieces < 7500 faces) on the
marching-cubes mesh of the BASELINE.json configs[2] stand-in — the 5,578-frame synthetic scan bench.py's `pipeline_c3` builds
(bench.make_sens_file), fused at 4 mm by scn_fuse_scene.  Reports V/F in and out, the GPU steps (CUDA events), the wall time of
scn_mesh_clean including the copies (best of 3 after a warm-up), the sequential C oracle on one thread beside them, and whether
the two agree bit for bit.  Then the rest of the decimate stage (DESIGN.md §6g): simplify.mlx twice on the cleaned mesh
(`_vh_clean.ply` -> `_vh_clean_1.ply` -> `_vh_clean_2.ply`), each call with its rounds, GPU phases, wall time including the copies
(best of 3 after a warm-up), V/F in and out, the one-thread decimation oracle and bit-identity (key "simplify").
Everything is written to a temporary directory; prints one JSON object.
Usage: python scripts/bench_meshclean.py [n_frames]"""
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 5578
    import torch
    import bench                                                # the stand-in scan generator; bench diverts stdout to stderr
    import meshclean_bindings as mb
    from scannet_b200 import fuse as sfuse
    from scannet_b200 import meshclean
    out = {"frames": n}
    with tempfile.TemporaryDirectory() as d:
        sens, ply = os.path.join(d, "scene.sens"), os.path.join(d, "scene_vh.ply")
        _, out["generate_s"] = bench.make_sens_file(sens, n, 7, torch.device("cuda:0"))
        sfuse.fuse_scene(sens, ply, max_blocks=1 << 22, hash_slots=1 << 24, decode_mode="gpu")
        xyz, rgb, tri = meshclean.load_rgb(ply)
    meshclean.clean(xyz, tri, rgb)                                                             # warm-up: module load, allocator
    walls, reps = [], []
    for _ in range(3):
        t0 = time.perf_counter()
        gx, gc, gt, rep = meshclean.clean(xyz, tri, rgb)
        walls.append(time.perf_counter() - t0); reps.append(rep)
    rep = reps[int(np.argmin(walls))]
    t0 = time.perf_counter()
    ox, oc, ot, cnt = mb.oracle_clean(xyz, tri, rgb)
    oracle_s = time.perf_counter() - t0
    out.update({k: rep[k] for k in ("vertices_in", "faces_in", "vertices_out", "faces_out") + tuple(mb.COUNTERS)})
    out["gpu_ms"] = {k: round(rep[k], 3) for k in ("upload_ms", "merge_ms", "dedup_ms", "pieces_ms", "download_ms")}
    out["wall_ms_incl_copies"] = round(min(walls) * 1e3, 3)
    out["wall_ms_runs"] = [round(w * 1e3, 3) for w in walls]
    out["oracle_1_thread_s"] = round(oracle_s, 3)
    out["bit_identical_to_oracle"] = (gx.tobytes() == ox.tobytes() and gc.tobytes() == oc.tobytes() and gt.tobytes() == ot.tobytes()
                                      and {k: rep[k] for k in mb.COUNTERS} == cnt)
    # simplify.mlx twice, each pass on the previous pass's output (the GPU's, which equals the oracle's when bit_identical)
    import meshsimplify_bindings as sb
    from scannet_b200 import meshsimplify
    sp, sa = meshsimplify.default_params()
    after = {"merge_threshold": sa.merge_threshold, "min_piece_faces": sa.min_piece_faces}
    passes = []
    x, c, t = gx, gc, gt
    for _ in range(2):
        meshsimplify.simplify(x, t, c, sp, sa)                                                 # warm-up
        walls, reps = [], []
        for _ in range(3):
            t0 = time.perf_counter()
            sx, sc, st, rep = meshsimplify.simplify(x, t, c, sp, sa)
            walls.append(time.perf_counter() - t0); reps.append(rep)
        rep = reps[int(np.argmin(walls))]
        t0 = time.perf_counter()
        ox, oc, ot, cnt, ccnt = sb.oracle_simplify(x, t, c, target_faces=sp.target_faces, target_perc=sp.target_perc,
                                                   quality_thr=sp.quality_thr, after=after)
        oracle_s = time.perf_counter() - t0
        d = {k: rep[k] for k in ("vertices_in", "faces_in", "vertices_out", "faces_out") + tuple(sb.COUNTERS)}
        d["gpu_ms"] = {k: round(rep[k], 3) for k in ("upload_ms", "quadrics_ms", "rounds_ms", "autoclean_ms", "clean_ms", "download_ms")}
        d["wall_ms_incl_copies"] = round(min(walls) * 1e3, 3)
        d["wall_ms_runs"] = [round(w * 1e3, 3) for w in walls]
        d["oracle_1_thread_s"] = round(oracle_s, 3)
        d["bit_identical_to_oracle"] = (sx.tobytes() == ox.tobytes() and sc.tobytes() == oc.tobytes() and st.tobytes() == ot.tobytes()
                                        and {k: rep[k] for k in sb.COUNTERS} == cnt and {k: rep["clean"][k] for k in mb.COUNTERS} == ccnt)
        passes.append(d)
        print(json.dumps(d), file=sys.stderr, flush=True)
        x, c, t = sx, sc, st
    out["simplify"] = passes
    bench.emit(out)


if __name__ == "__main__":
    main()
