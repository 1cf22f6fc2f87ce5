#!/usr/bin/env python
"""What a per-frame palette table costs the RGBA warp, against one table and against what callers did before it.

    python scripts/palette_perf.py [--steps 20] [--rounds 5] [--frames 16]

Workloads (bench.py's conventions: GPU-built lensmap, uniform random faces, CUDA events on the launch stream), each
into a view rectangle at (32, 16) of RGBA screens 64 pixels wider and 32 rows taller than the view:

    4k-cube-panini              f_fov 180, every pixel mapped
    4k-cube-fisheye1 (keep)     f_contain, about 44 % mapped, keep_unmapped
    4k-cube-quincuncial-rubix   f_cover + rubix; the gather kernel K3 runs in front of the ring kernel
    1080p-cube-panini170        f_fov 170

Microseconds per frame, for --frames-frame batches and for single-frame calls (frame f of the batch each time), of

    a  view_rgba                       one table for every frame (blinky_set_rgba_table)
    b  view_rgba_tables                frame f through tables[f] (blinky_warp_device_view_rgba_tables)
    c  set_rgba_table + 1-frame warp   today's workaround: per frame, replace the table, then warp that frame
    d  8-bit view + torch gather       an 8-bit warp, then tables[f][frame8] written into the RGBA screen

each the median over --rounds rounds of --steps calls.  Before timing, (b), (c) and (d) are checked byte for byte
against each other.  Prints one JSON line with the GPU's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench import WORKLOADS, setup_workload  # noqa: E402
from view_perf import gpu_identity  # noqa: E402

CASES = [("4k-cube-panini", False), ("4k-cube-fisheye1", True), ("4k-cube-quincuncial-rubix", False),
         ("1080p-cube-panini170", False)]
X0, Y0, PAD_X, PAD_Y = 32, 16, 64, 32


def smi_power_limit():
    """the enforced power limit as nvidia-smi reports it (a read-only query), for cards where NVML is not importable"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else None
    except (OSError, subprocess.SubprocessError, IndexError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()

    import torch

    import blinky_b200 as bb

    torch.cuda.set_device(0)
    sh = torch.cuda.current_stream().cuda_stream
    F = args.frames
    result = {"metric": "us_per_frame", "frames": F, "view_origin": [X0, Y0], "screen_pad": [PAD_X, PAD_Y],
              **gpu_identity(0), "nvidia_smi": smi_power_limit()}
    rows = []

    def timed(fn, frames_per_call):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        per_round = []
        for _ in range(args.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            per_round.append(e0.elapsed_time(e1) * 1e3 / (args.steps * frames_per_call))
        return round(float(np.median(per_round)), 2)

    for name, keep in CASES:
        W, H, PS = WORKLOADS[name][:3]
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        setup_workload(fe, name)
        fe.set_background(bb.synthetic_background(W, H))
        tables_np = np.random.default_rng(5).integers(0, 2**32, (F, 256), dtype=np.uint64).astype(np.uint32)
        tables = torch.from_numpy(tables_np.view(np.int32)).cuda()
        fe.set_rgba_table(tables_np[0])
        idx, _ = fe.lensmap()
        valid = torch.from_numpy(idx >= 0).cuda()
        gen = torch.Generator(device="cuda").manual_seed(1000)
        d_faces = torch.randint(0, 256, (F, fe.numplates, PS, PS), dtype=torch.uint8, device="cuda", generator=gen)
        SW, SH = W + PAD_X, H + PAD_Y
        screen = torch.zeros((F, SH, SW), dtype=torch.int32, device="cuda")
        screen8 = torch.zeros((F, SH, SW), dtype=torch.uint8, device="cuda")
        fill = torch.randint(-2**31, 2**31 - 1, (F, SH, SW), dtype=torch.int32, device="cuda", generator=gen)
        sview, sview8 = screen[:, Y0:Y0 + H, X0:X0 + W], screen8[:, Y0:Y0 + H, X0:X0 + W]
        offsets = (torch.arange(F, device="cuda", dtype=torch.int64) * 256).view(F, 1, 1)
        flat_tables = tables.reshape(-1)

        def view(frames, f0=0, **kw):
            fe.warp_view(d_faces[f0:f0 + frames], screen[f0:f0 + frames], x0=X0, y0=Y0, nframes=frames,
                         keep_unmapped=keep, rgba=True, stream=sh, **kw)

        def expand8(f0, frames):
            fe.warp_view(d_faces[f0:f0 + frames], screen8[f0:f0 + frames], x0=X0, y0=Y0, nframes=frames,
                         keep_unmapped=keep, stream=sh)
            rgba = flat_tables[sview8[f0:f0 + frames].to(torch.int64) + offsets[f0:f0 + frames]]
            dst = sview[f0:f0 + frames]
            dst.copy_(torch.where(valid, rgba, dst) if keep else rgba)

        batch = {
            "a": lambda: view(F),
            "b": lambda: view(F, tables=tables),
            "c": lambda: [(fe.set_rgba_table(tables_np[f]), view(1, f)) for f in range(F)],
            "d": lambda: expand8(0, F),
        }
        one_table = [tables[f:f + 1] for f in range(F)]   # (made once: a caller keeps its table tensors)
        single = {
            "a": lambda f: view(1, f),
            "b": lambda f: view(1, f, tables=one_table[f]),
            "c": lambda f: (fe.set_rgba_table(tables_np[f]), view(1, f)),
            "d": lambda f: expand8(f, 1),
        }
        # (b), (c) and (d) write the same screens
        outs, kernels = {}, {}
        for key in "bcd":
            screen.copy_(fill)
            batch[key]()
            torch.cuda.synchronize()
            outs[key] = screen.clone()
            kernels[key] = fe.last_kernel
        agree = bool(torch.equal(outs["b"], outs["c"]) and torch.equal(outs["b"], outs["d"]))
        del outs
        fe.set_rgba_table(tables_np[0])
        row = {"workload": name, "keep_unmapped": keep, "outputs_agree": agree}
        for key in "abcd":
            row[f"{key}_batch"] = timed(batch[key], F)
            if key in "ab":
                kernels[key] = fe.last_kernel
        counter = [0]

        def cycle(fn):
            def step():
                fn(counter[0] % F)
                counter[0] += 1
            return step

        for key in "abcd":
            row[f"{key}_single"] = timed(cycle(single[key]), 1)
        row["b_over_a_batch"] = round(row["b_batch"] / row["a_batch"], 4)
        row["b_over_a_single"] = round(row["b_single"] / row["a_single"], 4)
        row["kernels"] = kernels
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        del screen, screen8, fill, sview, sview8, d_faces
        fe.close()
        torch.cuda.empty_cache()
    result["results"] = rows
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
