"""Warp from a ray field turned by a per-frame matrix (blinky_warp_device_rays) against the loop it replaces, in one run.

At 3840x2160 on cube with 2048^2 plates, from the exported panini rays (f_fov 180):
  - the kernel per frame by CUDA events, 8-bit and RGBA, for 1 frame and batches of 8 and 16 frames sharing one field
    (ray_stride 0) with per-frame yaw matrices, and the bytes per second it reaches against the bytes it must move:
    the rays once per launch, the face sectors it samples (32-byte sectors per frame, counted from the lensmap of the
    same view) and the output;
  - a look-around frame: a 36-byte matrix upload plus the warp, to a device synchronise, eager and as a graph replay;
  - the existing loop: the field turned in torch, set_raymap_device, warp, to a device synchronise;
  - a small view in a large batch: 640x480, 64 frames sharing one field.
Prints one JSON line with the GPU's name, power limit and maximum SM clock.  Needs a GPU."""
import json
import os
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

    assert torch.cuda.is_available(), "ray_warp_perf needs a GPU"
    W, H, PS = 3840, 2160, 2048
    fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
    fe.command("f_globe cube")
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    fe.build_lensmap(W, H, PS, threads=0)
    d_rays = torch.empty((H, W, 3), dtype=torch.float32, device="cuda")
    fe.raymap(W, H, out=d_rays)
    torch.cuda.synchronize()
    nmax = 16
    xs = torch.from_numpy(np.stack([yaw(3.0 * i) for i in range(nmax)])).cuda()
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    out8 = torch.empty((nmax, H, W), dtype=torch.uint8, device="cuda")
    out32 = torch.empty((nmax, H, W), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    # bytes the kernel must move per launch: rays once, sampled 32-byte face sectors per frame, the output
    sectors = []
    rays_np, xs_np = d_rays.cpu().numpy(), xs.cpu().numpy()
    for i in range(nmax):
        fe.set_raymap(torch.from_numpy((rays_np @ xs_np[i].T).astype(np.float32)).cuda(), PS)
        m = fe.lensmap_packed().reshape(-1)
        idx = (m[(m & 0x80000000) != 0] & 0x0FFFFFFF).astype(np.int64)
        sectors.append(len(np.unique(idx // 32)) * 32)
    fe.set_raymap(d_rays, PS)
    ray_bytes = W * H * 12

    def time_kernel(rgba, n, reps=20):
        out = out32 if rgba else out8
        for _ in range(3):
            fe.warp_rays(d_faces, out, d_rays, xs[:n], nframes=n, rgba=rgba, face_stride=0, stream=st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fe.warp_rays(d_faces, out, d_rays, xs[:n], nframes=n, rgba=rgba, face_stride=0, stream=st)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        moved = ray_bytes + sum(sectors[:n]) + n * W * H * (4 if rgba else 1)
        return {"ms_per_launch": round(ms, 4), "ms_per_frame": round(ms / n, 4), "bytes_moved": moved, "GBps": round(moved / ms / 1e6, 1),
                "kernel": fe.last_kernel.split(" grid")[0]}

    res = {"size": f"{W}x{H}", "platesize": PS, "lens": "panini (exported rays)", "globe": "cube"}
    res.update(gpu_info())
    for rgba in (False, True):
        for n in (1, 8, 16):
            res[f"kernel_{'rgba' if rgba else '8bit'}_{n}"] = time_kernel(rgba, n)

    # a look-around frame: upload one matrix, warp, synchronise
    h_m = torch.from_numpy(yaw(10.0)).pin_memory()
    d_m = torch.empty((3, 3), dtype=torch.float32, device="cuda")
    one = out8[0]

    def frame():
        d_m.copy_(h_m, non_blocking=True)
        fe.warp_rays(d_faces, one, d_rays, d_m)
        torch.cuda.synchronize()

    def wall(fn, reps=100):
        for _ in range(5):
            fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return round((time.perf_counter() - t0) * 1e3 / reps, 4)

    res["look_around_eager_ms"] = wall(frame)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fe.warp_rays(d_faces, one, d_rays, d_m)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp_rays(d_faces, one, d_rays, d_m)

    def replay():
        d_m.copy_(h_m, non_blocking=True)
        g.replay()
        torch.cuda.synchronize()

    res["look_around_graph_ms"] = wall(replay)
    ref = one.clone()
    # the existing loop: torch turn, set_raymap_device, warp
    turned = torch.empty_like(d_rays)
    out_loop = torch.empty((H, W), dtype=torch.uint8, device="cuda")

    def loop():
        torch.matmul(d_rays, d_m.T, out=turned)
        fe.set_raymap(turned, PS)
        fe.warp(d_faces, out_loop, stream=st)
        torch.cuda.synchronize()

    res["existing_loop_ms"] = wall(loop, reps=20)
    res["loop_over_graph"] = round(res["existing_loop_ms"] / res["look_around_graph_ms"], 1)
    # the same frame both ways (the torch turn may round differently, so only the share of equal pixels is reported)
    res["loop_equal_pixel_share"] = round(float((out_loop == ref).float().mean().item()), 6)
    del g
    fe.release_captures()

    # a small view in a large batch (640x480, 64 frames, one shared field): the frames are split over rows of threads
    sw, sh, sn = 640, 480, 64
    fe.build_lensmap(sw, sh, PS, threads=0)
    s_rays = torch.empty((sh, sw, 3), dtype=torch.float32, device="cuda")
    fe.raymap(sw, sh, out=s_rays)
    s_xs = torch.from_numpy(np.stack([yaw(3.0 * i) for i in range(sn)])).cuda()
    s_out = torch.empty((sn, sh, sw), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        fe.warp_rays(d_faces, s_out, s_rays, s_xs, face_stride=0, stream=st)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        fe.warp_rays(d_faces, s_out, s_rays, s_xs, face_stride=0, stream=st)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    res[f"kernel_8bit_{sw}x{sh}_{sn}"] = {"ms_per_launch": round(ms, 4), "ms_per_frame": round(ms / sn, 4), "kernel": fe.last_kernel}
    fe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
