"""The ray export of forward-only lenses (blinky_get_raymap_forward_device, DESIGN §3h) at 3840x2160 on cube with
2048^2 plates, for sinusoidal, winkel1 and kavrayskiy7 at f_contain:
  - the first export call (the lens's NVRTC unit compiled) and the median of 5 repeat calls, host clock to return (the
    call returns with the field written);
  - fwd_ray_kernel alone, by the CUDA events around it that the export reports in blinky_build_info;
  - the median of 3 repeat blinky_build_lensmap(threads=0) builds of the same lens and size (the forward device build);
  - a look-around frame from the exported field: a 36-byte matrix upload plus warp_rays(filter="trilinear") with a
    persistent scratch, replayed as a CUDA graph, to a device synchronise (mean of 100).
Prints one JSON line with the GPU's name, power limit and maximum SM clock.  Needs a GPU."""
import json
import os
import re
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

    assert torch.cuda.is_available(), "raymap_forward_perf needs a GPU"
    W, H, PS = 3840, 2160, 2048
    fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
    fe.command("f_globe cube")
    d_faces = torch.from_numpy(bb.synthetic_faces(6, PS, 0)).cuda()
    field = torch.empty((H, W, 3), dtype=torch.float32, device="cuda")
    res = {"size": f"{W}x{H}", "platesize": PS, "globe": "cube", "zoom": "f_contain"}
    res.update(gpu_info())

    def export():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fe.raymap(W, H, out=field, forward=True, platesize=PS)
        ms = (time.perf_counter() - t0) * 1e3
        info = fe.build_info
        assert info.startswith("ray export (forward), device"), info
        return ms, float(re.search(r"\(rays ([0-9.]+) ms\)", info).group(1)), info

    for lens in ("sinusoidal", "winkel1", "kavrayskiy7"):
        fe.command(f"f_lens {lens}")
        fe.command("f_contain")
        first, _, first_info = export()
        repeat = [export() for _ in range(5)]
        builds = []
        for _ in range(4):
            t0 = time.perf_counter()
            fe.build_lensmap(W, H, PS, threads=0)
            builds.append((time.perf_counter() - t0) * 1e3)
        build_info = fe.build_info

        # a look-around frame from the exported field
        fe.raymap(W, H, out=field, forward=True, platesize=PS)
        fe.set_rgba_table(np.arange(256, dtype=np.uint32) * 0x01010101)
        out = torch.empty((H, W), dtype=torch.int32, device="cuda")
        scratch = torch.empty(fe.ray_pyramid_bytes(), dtype=torch.uint8, device="cuda")
        h_m = torch.from_numpy(yaw(10.0)).pin_memory()
        d_m = torch.empty((3, 3), dtype=torch.float32, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fe.warp_rays(d_faces, out, field, d_m, rgba=True, filter="trilinear", scratch=scratch)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fe.warp_rays(d_faces, out, field, d_m, rgba=True, filter="trilinear", scratch=scratch)

        def replay():
            d_m.copy_(h_m, non_blocking=True)
            g.replay()
            torch.cuda.synchronize()

        for _ in range(5):
            replay()
        t0 = time.perf_counter()
        for _ in range(100):
            replay()
        look = (time.perf_counter() - t0) * 1e3 / 100
        del g
        fe.release_captures()

        res[lens] = {"export_first_ms": round(first, 2), "export_repeat_ms": round(statistics.median(r[0] for r in repeat), 2),
                     "export_repeat_rounds_ms": [round(r[0], 2) for r in repeat],
                     "fwd_ray_kernel_ms": round(statistics.median(r[1] for r in repeat), 4),
                     "build_lensmap_repeat_ms": round(statistics.median(builds[1:]), 2), "build_rounds_ms": [round(b, 2) for b in builds],
                     "look_around_graph_trilinear_ms": round(look, 4), "first_export_info": first_info, "export_info": repeat[-1][2],
                     "build_info": build_info}
    fe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
