#!/usr/bin/env python
"""What a ray export costs at 4K (blinky_get_raymap_device), and a look-around frame that starts from it.

    python scripts/raymap_export_perf.py [--rounds 7] [--frames 60]

Screens of 3840x2160; lenses panini (f_fov 180), fisheye1 (f_contain), quincuncial (f_cover) and eckert4 (f_fov 180,
whose Newton loop flags about 8 % of the pixels in builds).  Per lens, medians over --rounds after one warm-up, host
clock unless named otherwise:

    first_call_ms     the first Fisheye.raymap into a CUDA tensor on a fresh context, to its return; nvrtc_ms is the
                      NVRTC compile of the ray-export unit inside it, as build_info reports it
    repeat_call_ms    the same call again (module cached)
    ray_kernel_ms     the ray-export kernel alone (CUDA events, from build_info)
    settled           pixels the interpreter evaluated (risk-flagged by the kernel)
    host_ms           Fisheye.raymap into host memory (the interpreter on all usable CPUs; host_threads)
    build_ms          a repeat build_lensmap(threads=0) of the same lens on cube with 2048^2 plates (module cached);
                      build_kernel_ms its lens kernel (CUDA events)

Then a look-around frame from exported panini rays on cube: a yaw in torch, set_raymap of the CUDA tensor, a 1-frame
8-bit warp, to the end of a device synchronise (look_around_ms, --frames frames), against a repeat
build_lensmap(threads=0) plus the same warp (rebuild_frame_ms).

Prints one JSON line with the GPU's name, power limit and maximum SM clock, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from supplied_perf import gpu_identity  # noqa: E402

W, H, PS = 3840, 2160, 2048
LENSES = [("panini", "f_fov 180"), ("fisheye1", "f_contain"), ("quincuncial", "f_cover"), ("eckert4", "f_fov 180")]


def median(xs):
    return round(statistics.median(xs), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--frames", type=int, default=60)
    args = ap.parse_args()

    import torch

    import blinky_b200 as bb

    assert torch.cuda.is_available(), "raymap_export_perf.py measures on the GPU"
    torch.cuda.set_device(0)
    clk = time.perf_counter

    def timed(call):
        torch.cuda.synchronize()
        t = clk()
        call()
        return (clk() - t) * 1e3

    def repeat(call):
        timed(call)
        return [timed(call) for _ in range(args.rounds)]

    result = {"metric": "host ms per 4K ray export (median)", **gpu_identity(), "rounds": args.rounds, "lenses": {}}
    d_rays = torch.empty((H, W, 3), dtype=torch.float32, device="cuda")
    for lens, zoom in LENSES:
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        fe.command("f_globe cube")
        fe.command(f"f_lens {lens}")
        fe.command(zoom)
        r = {"zoom": zoom}
        r["first_call_ms"] = round(timed(lambda: fe.raymap(W, H, out=d_rays)), 3)
        r["nvrtc_ms"] = float(re.search(r"NVRTC ([0-9.]+) ms", fe.build_info).group(1))
        calls, kernel = [], []
        timed(lambda: fe.raymap(W, H, out=d_rays))
        for _ in range(args.rounds):
            calls.append(timed(lambda: fe.raymap(W, H, out=d_rays)))
            kernel.append(float(re.search(r"kernel ([0-9.]+) ms", fe.build_info).group(1)))
        r["repeat_call_ms"] = median(calls)
        r["ray_kernel_ms"] = median(kernel)
        r["info"] = fe.build_info
        r["settled"] = int(fe.build_info.split("device: ")[1].split(" ")[0])
        r["host_ms"] = median(repeat(lambda: fe.raymap(W, H)))
        r["host_threads"] = len(os.sched_getaffinity(0))
        r["host_info"] = fe.build_info
        builds = repeat(lambda: fe.build_lensmap(W, H, PS, threads=0))
        r["build_ms"] = median(builds)
        r["build_info"] = fe.build_info
        r["build_kernel_ms"] = float(re.search(r"kernel ([0-9.]+) ms", fe.build_info).group(1))
        result["lenses"][lens] = r
        fe.close()

    fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
    fe.command("f_globe cube")
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    fe.raymap(W, H, out=d_rays)
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    d_out = torch.empty((H, W), dtype=torch.uint8, device="cuda")

    def frame(step):
        c, s = np.cos(0.01 * step), np.sin(0.01 * step)
        rot = torch.tensor([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=torch.float32, device="cuda")
        fe.set_raymap((d_rays @ rot.T).contiguous(), PS)
        fe.warp(d_faces, d_out, nframes=1)
        torch.cuda.synchronize()

    for s in range(3):
        frame(s)
    per = []
    for s in range(args.frames):
        t = clk()
        frame(s)
        per.append((clk() - t) * 1e3)
    look = {"look_around_ms": median(per), "look_around_info": fe.build_info}

    def rebuild():
        fe.build_lensmap(W, H, PS, threads=0)
        fe.warp(d_faces, d_out, nframes=1)
        torch.cuda.synchronize()

    look["rebuild_frame_ms"] = median(repeat(rebuild))
    look["rebuild_info"] = fe.build_info
    result["look_around"] = look
    fe.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
