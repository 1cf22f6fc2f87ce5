"""The trilinear RGBA warp from a ray field (blinky_warp_device_rays_trilinear) against the bilinear warp at k = 1 and
the supersampled warp at k = 2 and 4, alternated in one run.

At 3840x2160 on cube with 2048^2 plates, for three minifying fields — fisheye1 f_contain, equirect f_contain and panini
f_fov 180 — one field shared by every frame (exported at k*W x k*H for the supersampled warps) and 8 per-frame yaw
matrices per launch:
  - the kernel time by CUDA events over 20 launches after warm-up, every configuration alternated launch set by launch
    set and round by round (median of the rounds), in ms per frame; trilinear includes its pyramid launches;
  - the pyramid build alone: the same trilinear call with a 1 x 1 lensmap installed at the same plate size (the build
    does not depend on the view size);
  - a look-around frame: a 36-byte matrix upload plus the trilinear warp with a persistent scratch, replayed as a CUDA
    graph, to a device synchronise.
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

    assert torch.cuda.is_available(), "ray_trilinear_perf needs a GPU"
    W, H, PS = 3840, 2160, 2048
    n, reps, rounds = 8, 20, 3
    lenses = {"fisheye1_contain": ("fisheye1", "f_contain"), "equirect_contain": ("equirect", "f_contain"), "panini_fov180": ("panini", "f_fov 180")}
    configs = [("trilinear", 1), ("bilinear", 1), ("nearest", 2), ("nearest", 4)]
    fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
    fe.command("f_globe cube")
    fields = {}
    for tag, (lens, zoom) in lenses.items():
        fe.command(f"f_lens {lens}")
        fe.command(zoom)
        for k in sorted({k for _, k in configs}):
            fields[tag, k] = torch.empty((k * H, k * W, 3), dtype=torch.float32, device="cuda")
            fe.raymap(k * W, k * H, out=fields[tag, k])
    fe.build_lensmap(W, H, PS, threads=0)
    torch.cuda.synchronize()
    xs = torch.from_numpy(np.stack([yaw(3.0 * i) for i in range(n)])).cuda()
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    out = torch.empty((n, H, W), dtype=torch.int32, device="cuda")
    B = fe.ray_pyramid_bytes()
    scratch = torch.empty(n * B, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def launch(tag, filt, k):
        fe.warp_rays(d_faces, out, fields[tag, k], xs, nframes=n, rgba=True, face_stride=0, stream=st, supersample=k, filter=filt,
                     scratch=scratch if filt == "trilinear" else None)

    def time_kernel(fn):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    times = {(tag, f, k): [] for tag in lenses for f, k in configs}
    kernels = {}
    for _ in range(rounds):
        for tag in lenses:
            for f, k in configs:
                times[tag, f, k].append(time_kernel(lambda: launch(tag, f, k)))
                kernels[tag, f, k] = fe.last_kernel.split(" grid")[0]

    res = {"size": f"{W}x{H}", "platesize": PS, "globe": "cube", "frames_per_launch": n, "pyramid_bytes_per_frame": B,
           "fields": "one per lens, exported at k*W x k*H", "timing": f"CUDA events, {reps} launches after 3 warm-up, median of {rounds} rounds, "
                                                                     "all configurations alternated"}
    res.update(gpu_info())
    for (tag, f, k), ts in times.items():
        ms = statistics.median(ts)
        res[f"{tag}_{f}_k{k}"] = {"ms_per_frame": round(ms / n, 4), "rounds_ms_per_launch": [round(t, 4) for t in ts], "kernel": kernels[tag, f, k]}

    # the pyramid build alone: a 1 x 1 view at the same plate size
    small = torch.from_numpy(np.stack([fields["fisheye1_contain", 1][H // 2, W // 2].cpu().numpy()]).reshape(1, 1, 3)).cuda()
    fe.set_lensmap(np.full((1, 1), 0x70000000, np.uint32), PS, fe.numplates)
    one_px = torch.empty((n, 1, 1), dtype=torch.int32, device="cuda")
    ts = []
    for _ in range(rounds):
        ts.append(time_kernel(lambda: fe.warp_rays(d_faces, one_px, small, xs, nframes=n, rgba=True, face_stride=0, stream=st, filter="trilinear",
                                                   scratch=scratch)))
    res["pyramid_build_1x1_view"] = {"ms_per_frame": round(statistics.median(ts) / n, 4), "rounds_ms_per_launch": [round(t, 4) for t in ts],
                                     "launches": fe.last_kernel.split("levels=")[1]}
    fe.build_lensmap(W, H, PS, threads=0)

    # a look-around frame: upload one matrix, replay the captured trilinear warp, synchronise
    h_m = torch.from_numpy(yaw(10.0)).pin_memory()
    d_m = torch.empty((3, 3), dtype=torch.float32, device="cuda")
    one = out[0]
    field = fields["fisheye1_contain", 1]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fe.warp_rays(d_faces, one, field, d_m, rgba=True, filter="trilinear", scratch=scratch)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp_rays(d_faces, one, field, d_m, rgba=True, filter="trilinear", scratch=scratch)

    def replay():
        d_m.copy_(h_m, non_blocking=True)
        g.replay()
        torch.cuda.synchronize()

    for _ in range(5):
        replay()
    t0 = time.perf_counter()
    for _ in range(100):
        replay()
    res["look_around_graph_trilinear_ms"] = round((time.perf_counter() - t0) * 1e3 / 100, 4)
    del g
    fe.release_captures()
    fe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
