#!/usr/bin/env python
"""What a ray map costs at 4K (blinky_set_raymap_device).

    python scripts/raymap_perf.py [--rounds 9] [--frames 60]

Screens of 3840x2160 on the cube and `fast` globes with 2048^2 plates.  The rays are an equirectangular field made in
torch (the projection of the equirect lens, computed in float64 and narrowed to float32).  Reported per globe, medians
over --rounds after one warm-up, host clock unless named otherwise:

    first_call_ms        the first Fisheye.set_raymap of a CUDA tensor on a fresh context, to its return; nvrtc_ms is
                         the NVRTC compile of the ray-map unit inside it, as build_info reports it
    repeat_call_ms       the same call again (module cached); map_ms and plan_adopt_ms split it as build_info reports
                         (the ray pass with the interpreter's settling, then the GPU planner and the install)
    ray_kernel_ms        the ray kernel alone (CUDA events, from build_info)
    set_lensmap_ms       Fisheye.set_lensmap of the same packed map as a CUDA tensor (blinky_set_lensmap_device),
                         timed alternately with the repeat calls
    build_ms             a repeat build_lensmap(threads=0) of the equirect lens, f_contain (its module cached)
    look_around_ms       one frame of a look-around loop: the rays turned by a yaw in torch, set_raymap, and a 1-frame
                         8-bit warp, to the end of a device synchronise; --frames frames

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


def median(xs):
    return round(statistics.median(xs), 3)


def equirect(torch, yaw=0.0):
    y, x = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float64), torch.arange(W, device="cuda", dtype=torch.float64), indexing="ij")
    lon = (x / W - 0.5) * 2 * np.pi + yaw
    lat = (0.5 - y / H) * np.pi
    return torch.stack([torch.sin(lon) * torch.cos(lat), torch.sin(lat), torch.cos(lon) * torch.cos(lat)], -1).float().contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--frames", type=int, default=60)
    args = ap.parse_args()

    import torch

    import blinky_b200 as bb

    assert torch.cuda.is_available(), "raymap_perf.py measures on the GPU"
    torch.cuda.set_device(0)
    clk = time.perf_counter
    result = {"metric": "host ms per 4K ray map (median)", **gpu_identity(), "rounds": args.rounds, "globes": {}}
    rays = equirect(torch)
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    d_out = torch.empty((H, W), dtype=torch.uint8, device="cuda")
    for globe in ("cube", "fast"):
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        fe.command(f"f_globe {globe}")
        torch.cuda.synchronize()
        r = {}
        t0 = clk()
        fe.set_raymap(rays, PS)
        r["first_call_ms"] = round((clk() - t0) * 1e3, 3)
        r["nvrtc_ms"] = float(re.search(r"NVRTC ([0-9.]+) ms", fe.build_info).group(1))

        def timed(call):
            torch.cuda.synchronize()
            t = clk()
            call()
            return (clk() - t) * 1e3

        def repeat(call):
            timed(call)
            return [timed(call) for _ in range(args.rounds)]

        m = fe.lensmap_packed()
        d_map = torch.from_numpy(m.view(np.int32)).cuda()
        calls, kernel, map_ms, plan_ms, supplied = [], [], [], [], []
        timed(lambda: fe.set_raymap(rays, PS))
        timed(lambda: fe.set_lensmap(d_map, PS, fe.numplates))
        for _ in range(args.rounds):
            calls.append(timed(lambda: fe.set_raymap(rays, PS)))
            info = fe.build_info
            kernel.append(float(re.search(r"kernel ([0-9.]+) ms", info).group(1)))
            map_ms.append(float(re.search(r"map ([0-9.]+) ms", info).group(1)))
            plan_ms.append(float(re.search(r"plan\+adopt ([0-9.]+) ms", info).group(1)))
            supplied.append(timed(lambda: fe.set_lensmap(d_map, PS, fe.numplates)))
        r["repeat_call_ms"] = median(calls)
        r["map_ms"] = median(map_ms)
        r["plan_adopt_ms"] = median(plan_ms)
        r["ray_kernel_ms"] = median(kernel)
        r["set_lensmap_ms"] = median(supplied)
        fe.set_raymap(rays, PS)
        r["info"] = fe.build_info
        assert np.array_equal(fe.lensmap_packed(), m)
        fe.command("f_lens equirect")
        fe.command("f_contain")
        r["build_ms"] = median(repeat(lambda: fe.build_lensmap(W, H, PS, threads=0)))
        r["build_info"] = fe.build_info

        def frame(step):
            c, s = np.cos(0.01 * step), np.sin(0.01 * step)
            rot = torch.tensor([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=torch.float32, device="cuda")
            fe.set_raymap((rays @ rot.T).contiguous(), PS)
            fe.warp(d_faces[: fe.numplates], d_out, nframes=1)
            torch.cuda.synchronize()

        for s in range(3):
            frame(s)
        per = []
        for s in range(args.frames):
            t = clk()
            frame(s)
            per.append((clk() - t) * 1e3)
        r["look_around_ms"] = median(per)
        r["look_around_info"] = fe.build_info
        result["globes"][globe] = r
        fe.close()
        del d_map
    print(json.dumps(result))


if __name__ == "__main__":
    main()
