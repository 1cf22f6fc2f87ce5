#!/usr/bin/env python
"""What capturing the warp in a CUDA graph buys a host that warps one frame per call.

    python scripts/graph_perf.py [--calls 400] [--rounds 7] [--batch 16]

The in-engine shape: every call warps ONE frame, and the faces cycle through a device batch of --batch frames (the
faces miss L2, the tile plan stays resident).  Workloads (bench.py's conventions: GPU-built lensmap, uniform random
faces): 4K cube panini f_fov 180 and 1080p cube panini f_fov 170, each as an 8-bit dense frame
(blinky_warp_device) and as an RGBA view at (32, 16) of a screen 64 pixels wider and 32 rows taller
(blinky_warp_device_view_rgba).  Per workload:

    eager   one Fisheye.warp / warp_view call per frame
    graph   one torch.cuda.CUDAGraph per frame of the batch, each holding that frame's one-frame warp, replayed

Each is timed over --rounds rounds of --calls calls issued back to back on one stream: host microseconds per call
(the time to enqueue the calls, measured before the closing synchronise) and GPU microseconds per frame (CUDA events
around the calls), medians of the rounds.  Before timing, a replay of every graph is checked byte for byte against
the eager warp.  Prints one JSON line with the GPU's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, setup_workload  # noqa: E402

CASES = ["4k-cube-panini", "1080p-cube-panini170"]
X0, Y0, PAD_X, PAD_Y = 32, 16, 64, 32


def gpu_identity(index: int):
    import torch

    out = {"gpu": torch.cuda.get_device_name(index), "power_limit_w": "not measured"}
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        out["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception as e:  # noqa: BLE001
        out["nvml"] = f"unavailable: {e}"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()

    import torch

    import blinky_b200 as bb

    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    sh = stream.cuda_stream
    B = args.batch
    result = {"metric": "one-frame calls: host us per call, GPU us per frame", "batch": B, "calls": args.calls,
              "rounds": args.rounds, **gpu_identity(0)}
    rows = []

    def timed(call):
        """call(i) issues the i-th frame's work on `stream`: (host us per call, GPU us per frame), medians of rounds"""
        with torch.cuda.stream(stream):
            for i in range(args.warmup * B):
                call(i)
            torch.cuda.synchronize()
            host, gpu = [], []
            for _ in range(args.rounds):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                t0 = time.perf_counter()
                for i in range(args.calls):
                    call(i)
                t1 = time.perf_counter()
                e1.record(stream)
                torch.cuda.synchronize()
                host.append((t1 - t0) * 1e6 / args.calls)
                gpu.append(e0.elapsed_time(e1) * 1e3 / args.calls)
        return round(float(np.median(host)), 2), round(float(np.median(gpu)), 2)

    for name in CASES:
        W, H, PS = WORKLOADS[name][:3]
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        setup_workload(fe, name)
        fe.set_background(bb.synthetic_background(W, H))
        fe.set_rgba_table(np.random.default_rng(5).integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32))
        gen = torch.Generator(device="cuda").manual_seed(1000)
        d_faces = torch.randint(0, 256, (B, fe.numplates, PS, PS), dtype=torch.uint8, device="cuda", generator=gen)
        for rgba in (False, True):
            if rgba:
                screen = torch.zeros((H + PAD_Y, W + PAD_X), dtype=torch.int32, device="cuda")

                def warp(i, out=None):
                    fe.warp_view(d_faces[i % B], screen if out is None else out, x0=X0, y0=Y0, rgba=True, stream=sh)
            else:
                screen = torch.zeros((H, W), dtype=torch.uint8, device="cuda")

                def warp(i, out=None):
                    fe.warp(d_faces[i % B], screen if out is None else out, stream=sh)

            # the eager frames, then one graph per frame of the batch, each checked against its frame
            eager_out = [torch.zeros_like(screen) for _ in range(B)]
            with torch.cuda.stream(stream):
                for i in range(B):
                    warp(i, eager_out[i])
            torch.cuda.synchronize()
            graphs = []
            for i in range(B):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    fe.warp_view(d_faces[i], screen, x0=X0, y0=Y0, rgba=True) if rgba else fe.warp(d_faces[i], screen)
                graphs.append(g)
            agree = True
            for i in range(B):
                screen.zero_()
                graphs[i].replay()
                torch.cuda.synchronize()
                agree = agree and bool(torch.equal(screen, eager_out[i]))
            row = {"workload": name, "format": "rgba-view" if rgba else "8bit-dense", "graph_equals_eager": agree,
                   "kernel": fe.last_kernel}
            row["eager_host_us_per_call"], row["eager_gpu_us_per_frame"] = timed(warp)
            row["graph_host_us_per_call"], row["graph_gpu_us_per_frame"] = timed(lambda i: graphs[i % B].replay())
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del graphs, eager_out, screen
            fe.release_captures()
        fe.close()
        torch.cuda.empty_cache()
    result["results"] = rows
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
