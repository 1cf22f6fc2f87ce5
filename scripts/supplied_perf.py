#!/usr/bin/env python
"""What it costs to hand the warp a lensmap of one's own, at 4K.

    python scripts/supplied_perf.py [--rounds 7] [--frames 60]

Workloads: bench.py's 4K screens (3840x2160, cube globe of 6x2048^2 faces) with panini f_fov 180, fisheye1
f_contain and quincuncial f_cover with rubix.  Each lensmap is built once on the GPU, read back, and then handed in
again, timed with a host clock:

    device   Fisheye.set_lensmap of a CUDA tensor (blinky_set_lensmap_device: checked and planned on the GPU)
    pinned   Fisheye.set_lensmap of a numpy view of pinned host memory (blinky_set_lensmap: planned on host threads,
             then uploaded)
    build    a repeat build_lensmap(threads=0) of the same lens (the GPU lens evaluation; its NVRTC module is cached
             after the first build), with the `finish` and `plan+upload` steps build_info reports

Each is reported as the time from the call to its return, and to the end of the first 1-frame warp after it (the
warp enqueued right after the call, then a device synchronise), medians over --rounds rounds after one warm-up.

animated: --frames frames of a GPU-resident animation; each frame a small torch kernel rewrites the map (one zoom
step of a plate-0 magnifier), then set_lensmap (device) and a 1-frame RGBA warp; median host time per frame, from
the start of the map kernel to the end of the warp.

Prints one JSON line with the GPU's name and power limit, read in the same run.
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

from bench import WORKLOADS  # noqa: E402

CASES = {"panini": "4k-cube-panini", "fisheye1": "4k-cube-fisheye1", "quincuncial-rubix": "4k-cube-quincuncial-rubix"}


def gpu_identity():
    import subprocess

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": f"not read: {e}"}


def median(xs):
    return round(statistics.median(xs), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--frames", type=int, default=60)
    args = ap.parse_args()

    import torch

    import blinky_b200 as bb

    assert torch.cuda.is_available(), "supplied_perf.py measures on the GPU"
    torch.cuda.set_device(0)
    result = {"metric": "host ms per supplied 4K lensmap (median)", **gpu_identity(), "rounds": args.rounds, "cases": {}}
    clk = time.perf_counter
    for name, workload in CASES.items():
        W, H, PS, globe, lens, zoom, rubix = WORKLOADS[workload]
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        fe.command(f"f_globe {globe}")
        fe.command(f"f_lens {lens}")
        fe.command(zoom)
        fe.set_rubix(rubix)
        fe.build_lensmap(W, H, PS, threads=0)
        m = fe.lensmap_packed()
        n = fe.numplates
        d_map = torch.from_numpy(m.view(np.int32)).cuda()
        pinned_t = torch.from_numpy(m.view(np.int32)).pin_memory()
        pinned = pinned_t.numpy().view(np.uint32)
        d_faces = torch.from_numpy(bb.synthetic_faces(n, PS, 0)).cuda()
        d_out = torch.empty((H, W), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()

        def timed(call):
            t0 = clk()
            call()
            t1 = clk()
            fe.warp(d_faces, d_out, nframes=1)
            torch.cuda.synchronize()
            return (t1 - t0) * 1e3, (clk() - t0) * 1e3

        calls = {"device": lambda: fe.set_lensmap(d_map, PS, n), "pinned": lambda: fe.set_lensmap(pinned, PS, n),
                 "build": lambda: fe.build_lensmap(W, H, PS, threads=0)}
        case = {}
        for kind, call in calls.items():
            timed(call)   # warm-up
            ret, first, finish, plan_upload = [], [], [], []
            for _ in range(args.rounds):
                r, f = timed(call)
                ret.append(r)
                first.append(f)
                if kind == "build":
                    info = fe.build_info
                    finish.append(float(re.search(r"finish ([0-9.]+) ms", info).group(1)))
                    plan_upload.append(float(re.search(r"plan\+upload ([0-9.]+) ms", info).group(1)))
            case[kind] = {"call_ms": median(ret), "to_first_warp_ms": median(first)}
            if kind == "build":
                case[kind].update(finish_ms=median(finish), plan_upload_ms=median(plan_upload), info=fe.build_info)
            if kind == "device":
                case[kind]["info"] = fe.build_info
        # the three ways in give the same warp
        fe.set_lensmap(d_map, PS, n)
        assert np.array_equal(fe.lensmap_packed(), m)
        case["plan_summary"] = fe.plan_summary
        result["cases"][name] = case
        fe.close()
        del d_map, pinned_t, d_faces, d_out
        torch.cuda.empty_cache()

    # animated: a magnifier over plate 0 zooming in, one step per frame
    W, H, PS = 3840, 2160, 2048
    fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
    fe.command("f_globe cube")
    fe.set_rgba_table(np.arange(256, dtype=np.uint32) * 0x010101)
    y, x = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float32), torch.arange(W, device="cuda", dtype=torch.float32),
                          indexing="ij")
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    d_out = torch.empty((H, W), dtype=torch.int32, device="cuda")
    base = (0x80000000 | (7 << 28)) - 2**32   # valid, no tint, as int32

    def frame(step):
        z = 0.9 - 0.4 * (step % 60) / 60
        px = ((x - W / 2) * z * PS / W + PS / 2).to(torch.int32)
        py = ((y - H / 2) * z * PS / W + PS / 2).to(torch.int32)
        ok = (px >= 0) & (px < PS) & (py >= 0) & (py < PS)
        d_map = torch.where(ok, base + py * PS + px, torch.full_like(px, 7 << 28))
        fe.set_lensmap(d_map, PS, 6, stream=torch.cuda.current_stream().cuda_stream)
        fe.warp(d_faces, d_out, nframes=1, rgba=True)

    for s in range(3):
        frame(s)
    torch.cuda.synchronize()
    per = []
    for s in range(args.frames):
        t0 = clk()
        frame(s)
        torch.cuda.synchronize()
        per.append((clk() - t0) * 1e3)
    result["animated"] = {"frames": args.frames, "frame_ms": median(per), "frame_ms_min": round(min(per), 3), "info": fe.build_info}
    fe.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
