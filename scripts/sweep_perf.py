"""Developer sweep (run on the GPU machine): one process, many (environment knob, workload) combinations of the
device-resident warp; prints one line per combination.  Knobs are read when the context is created /
the lensmap is planned, so each combination gets a fresh context."""
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blinky_b200 as bb

WORK = {
    "panini": ("cube", "panini", "f_fov 180", 3840, 2160, 2048, False),
    "panini1080": ("cube", "panini", "f_fov 170", 1920, 1080, 1024, False),
    "quinc": ("cube", "quincuncial", "f_cover", 3840, 2160, 2048, True),
    "stereo": ("cube", "stereographic", "f_fov 180", 3840, 2160, 2048, False),
    "equirect": ("cube", "equirect", "f_contain", 3840, 2160, 2048, False),
    "hammer": ("cube", "hammer", "f_contain", 3840, 2160, 2048, False),
    "fisheye1": ("cube", "fisheye1", "f_contain", 3840, 2160, 2048, False),
    "trism": ("trism", "stereographic", "f_fov 180", 3840, 2160, 2048, False),
}
_faces = {}
_flush = None


def run(work, env, frames=16, iters=8, cold=False, kernel=0):
    global _flush
    g, l, z, W, H, PS, rubix = WORK[work]
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
        fe.command(f"f_globe {g}")
        fe.command(f"f_lens {l}")
        fe.command(z)
        if rubix:
            fe.command("f_rubix")
        fe.build_lensmap(W, H, PS, 0)
        fe.set_kernel(kernel)
        P = fe.numplates
        key = (P, PS, frames)
        if key not in _faces:
            gen = torch.Generator(device="cuda").manual_seed(1000)
            _faces.clear()
            _faces[key] = torch.randint(0, 256, (frames, P, PS, PS), dtype=torch.uint8, device="cuda", generator=gen)
        faces = _faces[key]
        out = torch.zeros((frames, H, W), dtype=torch.uint8, device="cuda")
        if _flush is None:
            _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        nf = 1 if cold else frames
        for _ in range(3):
            fe.warp(faces, out, nframes=nf, stream=st)
        torch.cuda.synchronize()
        times = []
        reps = 1 if cold else 10   # back-to-back launches between the events (as bench.py times them): no launch latency in the number
        for _ in range(iters):
            if cold:
                _flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fe.warp(faces, out, nframes=nf, stream=st)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) * 1e-3 / reps)
        t = float(np.median(times))
        print(json.dumps(dict(work=work, env=env, frames=nf, cold=cold, us_per_frame=round(t * 1e6 / nf, 2), min_us=round(min(times) * 1e6 / nf, 2),
                              tpx_s=round(W * H * nf / t / 1e12, 3), kernel=fe.last_kernel, plan=fe.plan_summary)), flush=True)
        fe.close()
    except Exception as ex:  # keep sweeping
        print(json.dumps(dict(work=work, env=env, error=str(ex)[:300])), flush=True)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


if __name__ == "__main__":
    # each argument: work[:cold][:k1][:fN],ENV=VAL,ENV=VAL
    for arg in sys.argv[1:]:
        parts = arg.split(",")
        head = parts[0].split(":")
        env = dict(p.split("=") for p in parts[1:] if p)
        frames = 16
        for h in head[1:]:
            if h.startswith("f"):
                frames = int(h[1:])
        run(head[0], env, frames=frames, cold="cold" in head[1:], kernel=1 if "k1" in head[1:] else 0)
