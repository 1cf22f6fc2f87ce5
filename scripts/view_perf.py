#!/usr/bin/env python
"""What writing into a view rectangle of a device screen costs, against what callers did before it existed.

    python scripts/view_perf.py [--steps 20] [--rounds 5] [--frames 16]

Workloads (bench.py's conventions: GPU-built lensmap, uniform random faces, 16-frame batches, CUDA events on the
launch stream): 4K cube panini f_fov 180 (every pixel mapped) and 4K cube fisheye1 f_contain (about 44 % mapped,
many EMPTY tiles), 8-bit and RGBA.  The screen is 64 pixels wider and 32 rows taller than the view, which sits at
(32, 16): an origin and pitch the fast kernels accept.  Per workload and pixel format, microseconds per frame of

    a  warp_device                     dense [H][W] frames
    b  warp_device_view, keep 0        into the screen, unmapped pixels get the background
    c  warp_device_view, keep 1        into the screen, only mapped pixels written
    d  a + cudaMemcpy2DAsync           dense frames, then one 2-D copy per frame into the screen
    e  a + masked merge                dense frames, then torch.where(valid, frame, screen) written into the screen

each the median over --rounds rounds of --steps launches.  Before timing, (b) is checked against (d) and (c)
against (e) byte for byte.  Prints one JSON line with the GPU's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, setup_workload  # noqa: E402

CASES = ["4k-cube-panini", "4k-cube-fisheye1"]
X0, Y0, PAD_X, PAD_Y = 32, 16, 64, 32


def cudart():
    """the CUDA runtime torch has loaded (for cudaMemcpy2DAsync, which torch does not expose)"""
    loaded = [line.split()[-1] for line in open("/proc/self/maps") if "libcudart.so" in line.split()[-1]]
    for path in loaded + ["libcudart.so.12", "libcudart.so"]:
        try:
            lib = ctypes.CDLL(path)
        except OSError:
            continue
        lib.cudaMemcpy2DAsync.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                          ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
        return lib
    raise RuntimeError("no CUDA runtime library found for cudaMemcpy2DAsync")


def gpu_identity(index: int):
    import torch

    out = {"gpu": torch.cuda.get_device_name(index), "power_limit_w": None}
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()

    import torch

    import blinky_b200 as bb

    torch.cuda.set_device(0)
    rt = cudart()
    stream = torch.cuda.current_stream()
    sh = stream.cuda_stream
    F = args.frames
    result = {"metric": "us_per_frame", "frames": F, "view_origin": [X0, Y0], "screen_pad": [PAD_X, PAD_Y], **gpu_identity(0)}
    rows = []

    def timed(fn):
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
            per_round.append(e0.elapsed_time(e1) * 1e3 / (args.steps * F))
        return round(float(np.median(per_round)), 2)

    for name in CASES:
        W, H, PS = WORKLOADS[name][:3]
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        setup_workload(fe, name)
        fe.set_background(bb.synthetic_background(W, H))
        fe.set_rgba_table(np.random.default_rng(5).integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32))
        idx, _ = fe.lensmap()
        valid = torch.from_numpy(idx >= 0).cuda()
        gen = torch.Generator(device="cuda").manual_seed(1000)
        d_faces = torch.randint(0, 256, (F, fe.numplates, PS, PS), dtype=torch.uint8, device="cuda", generator=gen)
        SW, SH = W + PAD_X, H + PAD_Y
        for rgba in (False, True):
            dt, bpp = (torch.int32, 4) if rgba else (torch.uint8, 1)
            dense = torch.zeros((F, H, W), dtype=dt, device="cuda")
            screen = torch.zeros((F, SH, SW), dtype=dt, device="cuda")
            fill = torch.randint(-2**31 if rgba else 0, 2**31 - 1 if rgba else 256, (F, SH, SW), dtype=dt, device="cuda", generator=gen)
            sview = screen[:, Y0:Y0 + H, X0:X0 + W]
            rowbytes, fstride = SW * bpp, SH * SW * bpp

            def a():
                fe.warp(d_faces, dense, nframes=F, rgba=rgba, stream=sh)

            def view(keep):
                return lambda: fe.warp_view(d_faces, screen, x0=X0, y0=Y0, nframes=F, keep_unmapped=keep, rgba=rgba, stream=sh)

            def d():
                a()
                origin = screen.data_ptr() + (Y0 * SW + X0) * bpp
                for f in range(F):
                    rc = rt.cudaMemcpy2DAsync(origin + f * fstride, rowbytes, dense[f].data_ptr(), W * bpp, W * bpp, H, 3, sh)
                    if rc != 0:
                        raise RuntimeError(f"cudaMemcpy2DAsync failed with {rc}")

            def e():
                a()
                sview.copy_(torch.where(valid, dense, sview))

            # the view calls give what the two-pass versions give
            outs = {}
            for key, fn in (("b", view(False)), ("d", d), ("c", view(True)), ("e", e)):
                screen.copy_(fill)
                fn()
                torch.cuda.synchronize()
                outs[key] = screen.clone()
            agree = bool(torch.equal(outs["b"], outs["d"]) and torch.equal(outs["c"], outs["e"]))
            kernels = {}
            row = {"workload": name, "format": "rgba" if rgba else "8bit", "mapped_frac": round(float(valid.float().mean()), 3),
                   "outputs_agree": agree}
            for key, fn in (("a_dense", a), ("b_view", view(False)), ("c_view_keep", view(True)), ("d_dense_memcpy2d", d),
                            ("e_dense_masked_merge", e)):
                row[key] = timed(fn)
                if key[0] in "abc":
                    kernels[key[0]] = fe.last_kernel
            row["kernels"] = kernels
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del dense, screen, fill, sview, outs
        fe.close()
        torch.cuda.empty_cache()
    result["results"] = rows
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
