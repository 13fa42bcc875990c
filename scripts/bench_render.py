#!/usr/bin/env python
"""Render benchmark (DESIGN.md §6i): the `render` stage on the `_vh_clean_2` mesh of the BASELINE.json configs[2] stand-in,
built as scripts/bench_meshclean.py builds its meshes (bench.make_sens_file, scn_fuse_scene at 4 mm, clean.mlx, simplify.mlx
twice).  Times the script's default single view (640x480, 16 spp, path) and its 72-view turntable: PLY load, BVH build and
trace (CUDA events), PNG encode + write, rays/s, best of 3 after a warm-up.  The oracle renders a sample of 16x16 pixel tiles
of the single view (labelled as sampled) and the result says whether they are bit-identical.  Card name, power limit and SM
clock are read in the same call.  Ray tracing is bound neither by bandwidth nor by FLOPs in a way a data-sheet peak
describes, so rays/s and the counters are reported, not a share of peak.  Everything is written to a temporary directory;
prints one JSON object.
Usage: python scripts/bench_render.py [n_frames]"""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "unavailable"


def timed_render(xyz, rgb, tri, p, cams, render):
    render.render(xyz, rgb, tri, p, cams)                                                   # warm-up
    runs = []
    for _ in range(3):
        t0 = time.perf_counter()
        img, rep = render.render(xyz, rgb, tri, p, cams)
        runs.append((time.perf_counter() - t0, rep, img))
    wall, rep, img = min(runs, key=lambda r: r[0])
    rays = rep["primary_rays"] + rep["secondary_rays"]
    d = {k: rep[k] for k in ("views", "pixels", "samples", "primary_rays", "secondary_rays", "primary_hits", "node_visits",
                             "triangle_tests", "bvh_nodes")}
    d["gpu_ms"] = {k: round(rep[k], 3) for k in ("upload_ms", "bvh_ms", "trace_ms", "download_ms")}
    d["wall_ms"] = round(wall * 1e3, 3)
    d["wall_ms_runs"] = [round(r[0] * 1e3, 3) for r in runs]
    d["rays_per_s_trace"] = round(rays / (rep["trace_ms"] * 1e-3), 1)
    d["node_visits_per_ray"] = round(rep["node_visits"] / rays, 2)
    d["triangle_tests_per_ray"] = round(rep["triangle_tests"] / rays, 2)
    return d, img


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1500
    import torch
    import bench                                                # the stand-in scan generator; bench diverts stdout to stderr
    import render_bindings as rb
    from scannet_b200 import fuse as sfuse
    from scannet_b200 import meshclean, meshsimplify, render
    out = {"frames": n, "gpu": gpu_info()}
    with tempfile.TemporaryDirectory() as d:
        sens, ply = os.path.join(d, "scene.sens"), os.path.join(d, "scene_vh.ply")
        _, out["generate_s"] = bench.make_sens_file(sens, n, 7, torch.device("cuda:0"))
        sfuse.fuse_scene(sens, ply, max_blocks=1 << 22, hash_slots=1 << 24, decode_mode="gpu")
        xyz, rgb, tri = meshclean.load_rgb(ply)
        x, c, t, _ = meshclean.clean(xyz, tri, rgb)
        sp, sa = meshsimplify.default_params()
        for _ in range(2):
            x, c, t, _ = meshsimplify.simplify(x, t, c, sp, sa)
        mesh = os.path.join(d, "scene_vh_clean_2.ply")
        from scannet_b200._lib import check, lib
        import ctypes as C
        x = np.ascontiguousarray(x); c = np.ascontiguousarray(c); t = np.ascontiguousarray(t)
        check(lib().scn_mesh_save_ply(mesh.encode(), x.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p), C.c_uint64(len(x)),
                                  t.ctypes.data_as(C.c_void_p), C.c_uint64(len(t))))
        t0 = time.perf_counter()
        xyz, rgb, tri = meshclean.load_rgb(mesh)
        out["load_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
        out["mesh"] = {"vertices": len(xyz), "faces": len(tri)}
        p = render.default_params()
        single, img = timed_render(xyz, rgb, tri, p, [render.camera(xyz, p)], render)
        # the CLI end to end: its output line has the BVH, trace and PNG encode + write times
        t0 = time.perf_counter()
        r = subprocess.run([os.path.join(ROOT, "scannet_b200/bin/render"), mesh], capture_output=True, text=True)
        single["cli_wall_s"] = round(time.perf_counter() - t0, 3)
        single["cli_ok"] = r.returncode == 0 and os.path.exists(os.path.join(d, "scene_vh_clean_2.png"))
        single["cli_output"] = r.stdout.strip()
        from PIL import Image
        single["cli_png_matches_library"] = bool(single["cli_ok"] and
                                                 np.array(Image.open(os.path.join(d, "scene_vh_clean_2.png"))).tobytes() == img[0].tobytes())
        out["single_view"] = single
        print(json.dumps(single), file=sys.stderr, flush=True)
        cams = [render.camera(xyz, p, a, turntable=True) for a in render.turntable_angles(5)]
        turn, _ = timed_render(xyz, rgb, tri, p, cams, render)
        t0 = time.perf_counter()
        r = subprocess.run([os.path.join(ROOT, "scannet_b200/bin/render"), "--render_turntable", mesh], capture_output=True, text=True)
        turn["cli_wall_s"] = round(time.perf_counter() - t0, 3)
        turn["cli_output"] = r.stdout.strip()
        turn["cli_frames_written"] = sum(os.path.exists(nm) for nm in render.turntable_names(mesh, 5))
        out["turntable"] = turn
        print(json.dumps(turn), file=sys.stderr, flush=True)
        # the oracle on sampled 16x16 tiles of the single view
        rng = np.random.default_rng(0)
        tiles = [(int(rng.integers(0, p.width // 16)) * 16, int(rng.integers(0, p.height // 16)) * 16) for _ in range(12)]
        cam = [render.camera(xyz, p)]
        same = True
        t0 = time.perf_counter()
        for tx, ty in tiles:
            o, _ = rb.oracle_render(xyz, rgb, tri, p, cam, mode=1, rect=(tx, ty, 16, 16))
            same &= o[0].tobytes() == img[0, ty:ty + 16, tx:tx + 16].tobytes()
        out["oracle_sampled_tiles"] = {"tiles": len(tiles), "size": 16, "seconds": round(time.perf_counter() - t0, 3),
                                       "threads": os.cpu_count(), "bit_identical": bool(same)}
    out["gpu_after"] = gpu_info()
    bench.emit(out)


if __name__ == "__main__":
    main()
