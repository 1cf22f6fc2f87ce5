"""The supersampled RGBA warp from a ray field (blinky_warp_device_rays_supersampled) against the one-sample RGBA ray warp,
interleaved in one run.

At 3840x2160 on cube with 2048^2 plates, from the panini rays (f_fov 180) exported at k*W x k*H, one field shared by
every frame and per-frame yaw matrices:
  - the kernel by CUDA events over 20 launches after warm-up, for k = 1 (warp_rays, rgba=True), 2, 3 and 4 and batches
    of 1 and 8 frames, the configurations interleaved round by round (median of the rounds); ms per frame, samples
    (rays) per second and the field bytes one launch reads (12 * k^2 * W * H);
  - a look-around frame at k = 2: a 36-byte matrix upload plus the warp, replayed as a CUDA graph, to a device
    synchronise.
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

    assert torch.cuda.is_available(), "ray_supersample_perf needs a GPU"
    W, H, PS = 3840, 2160, 2048
    factors, batches, reps, rounds = (1, 2, 3, 4), (1, 8), 20, 5
    fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
    fe.command("f_globe cube")
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    fields = {}
    for k in factors:
        fields[k] = torch.empty((k * H, k * W, 3), dtype=torch.float32, device="cuda")
        fe.raymap(k * W, k * H, out=fields[k])
    fe.build_lensmap(W, H, PS, threads=0)
    torch.cuda.synchronize()
    nmax = max(batches)
    xs = torch.from_numpy(np.stack([yaw(3.0 * i) for i in range(nmax)])).cuda()
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    out = torch.empty((nmax, H, W), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def launch(k, n):
        fe.warp_rays(d_faces, out, fields[k], xs[:n], nframes=n, rgba=True, face_stride=0, stream=st, supersample=k)

    def time_kernel(k, n):
        for _ in range(3):
            launch(k, n)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            launch(k, n)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    times = {(k, n): [] for k in factors for n in batches}
    kernels = {}
    for _ in range(rounds):
        for n in batches:
            for k in factors:
                times[(k, n)].append(time_kernel(k, n))
                kernels[(k, n)] = fe.last_kernel.split(" block")[0]

    res = {"size": f"{W}x{H}", "platesize": PS, "lens": "panini f_fov 180 (exported at k*W x k*H)", "globe": "cube",
           "timing": f"CUDA events, {reps} launches after 3 warm-up, median of {rounds} interleaved rounds"}
    res.update(gpu_info())
    for (k, n), ts in times.items():
        ms = statistics.median(ts)
        res[f"k{k}_frames{n}"] = {"ms_per_launch": round(ms, 4), "ms_per_frame": round(ms / n, 4),
                                  "rounds_ms": [round(t, 4) for t in ts],
                                  "gsamples_per_s": round(k * k * W * H * n / ms / 1e6, 2),
                                  "field_bytes_per_launch": 12 * k * k * W * H, "kernel": kernels[(k, n)]}

    # a look-around frame at k = 2: upload one matrix, replay the captured warp, synchronise
    h_m = torch.from_numpy(yaw(10.0)).pin_memory()
    d_m = torch.empty((3, 3), dtype=torch.float32, device="cuda")
    one = out[0]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fe.warp_rays(d_faces, one, fields[2], d_m, rgba=True, supersample=2)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp_rays(d_faces, one, fields[2], d_m, rgba=True, supersample=2)

    def replay():
        d_m.copy_(h_m, non_blocking=True)
        g.replay()
        torch.cuda.synchronize()

    for _ in range(5):
        replay()
    t0 = time.perf_counter()
    for _ in range(100):
        replay()
    res["look_around_graph_k2_ms"] = round((time.perf_counter() - t0) * 1e3 / 100, 4)
    del g
    fe.release_captures()
    fe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
