"""PCIe reality check for the end-to-end path: what do H2D and D2H reach together, and what
does blinky_warp_host reach on a 4K panini batch?"""
import os, sys, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch

def bw(nbytes_h2d, nbytes_d2h, reps=30):
    h_in = torch.empty(nbytes_h2d or 1, dtype=torch.uint8).pin_memory()
    d_in = torch.empty(nbytes_h2d or 1, dtype=torch.uint8, device="cuda")
    h_out = torch.empty(nbytes_d2h or 1, dtype=torch.uint8).pin_memory()
    d_out = torch.empty(nbytes_d2h or 1, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    def run():
        if nbytes_h2d:
            with torch.cuda.stream(s1): d_in.copy_(h_in, non_blocking=True)
        if nbytes_d2h:
            with torch.cuda.stream(s2): h_out.copy_(d_out, non_blocking=True)
    for _ in range(3): run()
    torch.cuda.synchronize(); t = time.perf_counter()
    for _ in range(reps): run()
    torch.cuda.synchronize(); dt = (time.perf_counter() - t) / reps
    return nbytes_h2d / dt / 1e9, nbytes_d2h / dt / 1e9

for a, b in [(64 << 20, 64 << 20)]:
    h, d = bw(a, b)
    print(f"H2D {a>>20:3d} MiB + D2H {b>>20:3d} MiB per round: H2D {h:6.1f} GB/s  D2H {d:6.1f} GB/s", flush=True)

import blinky_b200 as bb
W, H, PS, F = 3840, 2160, 2048, 16
fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
for c in ("f_globe cube", "f_lens panini", "f_fov 180"): fe.command(c)
fe.build_lensmap(W, H, PS, threads=0)
faces = fe.alloc_pinned(F * 6 * PS * PS).reshape(F, -1); faces[:] = np.random.default_rng(0).integers(0, 256, faces.shape, dtype=np.uint8)
out = fe.alloc_pinned(F * W * H).reshape(F, H, W)
for _ in range(2): fe.warp_host(faces, dst=out)
t = time.perf_counter(); n = 4
for _ in range(n): fe.warp_host(faces, dst=out)
dt = (time.perf_counter() - t) / n
want = fe.warp_host(faces[:2].copy(), keep_unmapped=False)
assert np.array_equal(want, out[:2]), "pinned and pageable buffers give different frames"
print(json.dumps({"ms_per_frame": dt / F * 1e3, "gpx_s": W * H * F / dt / 1e9,
                  "h2d_gbs": fe.upload_bytes_per_frame * F / dt / 1e9, "d2h_gbs": W * H * F / dt / 1e9}))
