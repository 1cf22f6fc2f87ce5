#!/usr/bin/env python
"""What warping straight from a 3x2 atlas costs, against dense faces and against repacking the atlas first.

    python scripts/layout_perf.py [--steps 20] [--rounds 5] [--frames 16]

Workloads (bench.py's conventions: GPU-built lensmap, uniform random faces, CUDA events on the launch stream):
4k-cube-panini, 4k-cube-fisheye1 (f_contain), 4k-cube-quincuncial-rubix (f_cover + rubix) and 1080p-cube-panini170,
each in 8-bit and RGBA.  The atlas holds the six plates in a 3x2 grid with 16-byte gaps, rows padded to a multiple of
16 bytes plus 16.  Microseconds per frame, for --frames-frame batches and for single-frame calls, of

    a  dense        the warp of contiguous [frame][plate][ps][ps] faces
    b  layout       the same warp reading the atlas through blinky_set_face_layout
    c  repack       torch copies the atlas into contiguous faces, then the dense warp
    d  stacked      the contiguous faces read through a layout that describes them (rowbytes = ps, plate i at row
                    i * ps): the layout's addressing alone, without the atlas's longer rows

each the median over --rounds rounds of --steps calls.  (a) to (d) are checked byte for byte against each other
first.  Prints one JSON line with the GPU's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench import WORKLOADS, setup_workload  # noqa: E402
from palette_perf import smi_power_limit  # noqa: E402
from view_perf import gpu_identity  # noqa: E402

CASES = ["4k-cube-panini", "4k-cube-fisheye1", "4k-cube-quincuncial-rubix", "1080p-cube-panini170"]


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
    result = {"metric": "us_per_frame", "frames": F, **gpu_identity(0), "nvidia_smi": smi_power_limit()}
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

    for name in CASES:
        W, H, PS = WORKLOADS[name][:3]
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        setup_workload(fe, name)
        fe.set_background(bb.synthetic_background(W, H))
        P = fe.numplates
        gap = 16
        origins = [(c * (PS + gap), r * (PS + gap)) for r in range(2) for c in range(3)][:P]
        rowbytes = -(-(3 * PS + 2 * gap) // 16) * 16 + 16
        rows_n = 2 * PS + gap
        gen = torch.Generator(device="cuda").manual_seed(1000)
        atlas = torch.randint(0, 256, (F, rows_n, rowbytes), dtype=torch.uint8, device="cuda", generator=gen)
        dense = torch.empty((F, P, PS, PS), dtype=torch.uint8, device="cuda")
        for i, (x, y) in enumerate(origins):
            dense[:, i] = atlas[:, y:y + PS, x:x + PS]
        repacked = torch.empty_like(dense)
        for rgba in (False, True):
            out = torch.empty((F, H, W * (4 if rgba else 1)), dtype=torch.uint8, device="cuda")

            def warp(faces, frames, f0=0, face_stride=None):
                fe.warp(faces[f0:f0 + frames], out[f0:f0 + frames], nframes=frames, rgba=rgba, stream=sh, face_stride=face_stride)

            def repack(frames, f0=0):
                for i, (x, y) in enumerate(origins):
                    repacked[f0:f0 + frames, i].copy_(atlas[f0:f0 + frames, y:y + PS, x:x + PS])
                warp(repacked, frames, f0)

            fns = {"a": lambda frames, f0=0: warp(dense, frames, f0),
                   "b": lambda frames, f0=0: warp(atlas, frames, f0),
                   "c": repack,
                   "d": lambda frames, f0=0: warp(dense, frames, f0, face_stride=P * PS * PS)}
            # the context's face layout while each variant runs (set once, outside the timed calls)
            layouts = {"a": None, "b": (rowbytes, origins), "c": None, "d": (PS, [(0, i * PS) for i in range(P)])}

            def use(key):
                if layouts[key]:
                    fe.set_face_layout(*layouts[key])
                else:
                    fe.set_face_layout()

            outs, kernels = {}, {}
            for key in "abcd":
                use(key)
                out.zero_()
                fns[key](F)
                torch.cuda.synchronize()
                outs[key] = out.clone()
                kernels[key] = fe.last_kernel
            agree = all(torch.equal(outs["a"], outs[k]) for k in "bcd")
            del outs
            row = {"workload": name, "rgba": rgba, "outputs_agree": agree, "rowbytes": rowbytes}
            counter = [0]

            def cycle(fn):
                def step():
                    fn(1, counter[0] % F)
                    counter[0] += 1
                return step

            for key in "abcd":
                use(key)
                row[f"{key}_batch"] = timed(lambda: fns[key](F), F)
                row[f"{key}_single"] = timed(cycle(fns[key]), 1)
            fe.set_face_layout()
            row["b_over_a_batch"] = round(row["b_batch"] / row["a_batch"], 4)
            row["b_over_a_single"] = round(row["b_single"] / row["a_single"], 4)
            row["kernels"] = kernels
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del out
        del atlas, dense, repacked
        fe.close()
        torch.cuda.empty_cache()
    result["results"] = rows
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
