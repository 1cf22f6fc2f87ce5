"""The bilinear RGBA warp from a ray field (blinky_warp_device_rays_bilinear) against the nearest RGBA ray warps at the same
factor (blinky_warp_device_rays_rgba at k = 1, blinky_warp_device_rays_supersampled at k = 2..4), alternated in one run.

At 3840x2160 on cube with 2048^2 plates, for two fields exported at k*W x k*H — rectilinear f_fov 75 (the plates
magnified over most of the view) and panini f_fov 180 (minified at the edges) — one field shared by every frame and 8
per-frame yaw matrices per launch:
  - the kernel by CUDA events over 20 launches after warm-up, for k = 1, 2, 3 and 4, bilinear and nearest alternated
    launch set by launch set and round by round (median of the rounds); ms per frame and samples per second;
  - a look-around frame at k = 1: a 36-byte matrix upload plus the bilinear warp, replayed as a CUDA graph, to a
    device synchronise.
Prints one JSON line with the GPU's name, power limit and maximum SM clock.  Needs a GPU."""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import blinky_b200 as bb  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "error": str(e)}


def yaw(deg):
    a = np.radians(deg)
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32)


def main():
    import torch

    assert torch.cuda.is_available(), "ray_bilinear_perf needs a GPU"
    W, H, PS = 3840, 2160, 2048
    factors, n, reps, rounds = (1, 2, 3, 4), 8, 20, 3
    lenses = {"rectilinear_fov75": ("rectilinear", 75), "panini_fov180": ("panini", 180)}
    fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
    fe.command("f_globe cube")
    fields = {}
    for tag, (lens, fov) in lenses.items():
        fe.command(f"f_lens {lens}")
        fe.command(f"f_fov {fov}")
        for k in factors:
            fields[tag, k] = torch.empty((k * H, k * W, 3), dtype=torch.float32, device="cuda")
            fe.raymap(k * W, k * H, out=fields[tag, k])
    fe.build_lensmap(W, H, PS, threads=0)
    torch.cuda.synchronize()
    xs = torch.from_numpy(np.stack([yaw(3.0 * i) for i in range(n)])).cuda()
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    out = torch.empty((n, H, W), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def launch(tag, k, filt):
        fe.warp_rays(d_faces, out, fields[tag, k], xs, nframes=n, rgba=True, face_stride=0, stream=st, supersample=k, filter=filt)

    def time_kernel(tag, k, filt):
        for _ in range(3):
            launch(tag, k, filt)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            launch(tag, k, filt)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    filters = ("bilinear", "nearest")
    times = {(tag, k, f): [] for tag in lenses for k in factors for f in filters}
    kernels = {}
    for _ in range(rounds):
        for tag in lenses:
            for k in factors:
                for f in filters:
                    times[tag, k, f].append(time_kernel(tag, k, f))
                    kernels[tag, k, f] = fe.last_kernel.split(" grid")[0]

    res = {"size": f"{W}x{H}", "platesize": PS, "globe": "cube", "frames_per_launch": n, "fields": "one per lens, exported at k*W x k*H",
           "timing": f"CUDA events, {reps} launches after 3 warm-up, median of {rounds} rounds, bilinear and nearest alternated"}
    res.update(gpu_info())
    for (tag, k, f), ts in times.items():
        ms = statistics.median(ts)
        res[f"{tag}_k{k}_{f}"] = {"ms_per_frame": round(ms / n, 4), "rounds_ms_per_launch": [round(t, 4) for t in ts],
                                  "gsamples_per_s": round(k * k * W * H * n / ms / 1e6, 2), "kernel": kernels[tag, k, f]}

    # a look-around frame at k = 1: upload one matrix, replay the captured bilinear warp, synchronise
    h_m = torch.from_numpy(yaw(10.0)).pin_memory()
    d_m = torch.empty((3, 3), dtype=torch.float32, device="cuda")
    one = out[0]
    field = fields["rectilinear_fov75", 1]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fe.warp_rays(d_faces, one, field, d_m, rgba=True, filter="bilinear")
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp_rays(d_faces, one, field, d_m, rgba=True, filter="bilinear")

    def replay():
        d_m.copy_(h_m, non_blocking=True)
        g.replay()
        torch.cuda.synchronize()

    for _ in range(5):
        replay()
    t0 = time.perf_counter()
    for _ in range(100):
        replay()
    res["look_around_graph_k1_bilinear_ms"] = round((time.perf_counter() - t0) * 1e3 / 100, 4)
    del g
    fe.release_captures()
    fe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
