"""Warps from faces laid out in a pitched surface (blinky_set_face_layout), on the GPU.

Every output byte is compared with the dense warp of the same faces, which the rest of the suite pins to the oracle;
8-bit single frames are also compared with the CPU oracle directly.  Surfaces are filled with random bytes before the
plates are placed, so a kernel that read a gap texel into a pixel would show; the gap-independence checks refill the
gaps with other bytes and expect the same output."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch

    return torch


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


def setup(fe, globe, lens, zoom, size, rubix):
    W, H, PS = size
    fe.command(f"f_globe {globe}")
    fe.command(f"f_lens {lens}")
    if zoom:
        fe.command(zoom)
    fe.set_rubix(rubix)
    fe.build_lensmap(W, H, PS, 8)


def r16(v):
    return -(-v // 16) * 16


def layouts(ps, n):
    """name -> (rowbytes, origins, rows, kernel the ring-kernel-eligible dense warp becomes)"""
    atlas = [(c * (ps + 16), r * (ps + 9)) for r in range(2) for c in range(3)]
    odd = [(c * (ps + 5) + 3, r * (ps + 7) + 1) for r in range(2) for c in range(3)]
    return {
        "dense-equivalent": (ps, [(0, i * ps) for i in range(n)], n * ps, "warp_ring_kernel"),
        "stacked-padded": (ps + 48, [(16, i * (ps + 5) + 2) for i in range(n)], n * (ps + 5) + 2 + 3, "warp_ring_kernel"),
        "atlas-3x2": (r16(3 * ps + 32 + 1), atlas[:n], 2 * ps + 9, "warp_ring_kernel"),
        "odd-origins": (r16(3 * ps + 13), odd[:n], 2 * ps + 8, "warp_gather_kernel"),
        "odd-pitch": (3 * ps + 32 + 7, atlas[:n], 2 * ps + 9, "warp_gather_kernel"),
    }


def surfaces(faces, rowbytes, origins, rows, seed):
    """[N, rows, rowbytes] random bytes with plate i of each frame at origins[i]"""
    n, p, ps, _ = faces.shape
    out = np.random.default_rng(seed).integers(0, 256, (n, rows, rowbytes), dtype=np.uint8)
    for i in range(p):
        x, y = origins[i]
        out[:, y:y + ps, x:x + ps] = faces[:, i]
    return out


def faces_batch(bb, fe, n, seed):
    return np.stack([bb.synthetic_faces(fe.numplates, fe.platesize, seed + i) for i in range(n)])


def run(torch, fe, d_faces, nframes, mode, tables=None):
    """one warp into a sentinel-filled buffer: "8bit", "rgba", "tables" (RGBA, per-frame tables), "view-keep"
    (8-bit view rectangle, only mapped pixels written); returns the buffer on the host"""
    W, H = fe.width, fe.height
    if mode == "view-keep":
        screen = torch.full((nframes, H + 5, W + 24), 0x5A, dtype=torch.uint8, device="cuda")
        fe.warp_view(d_faces, screen, x0=8, y0=3, nframes=nframes, keep_unmapped=True)
    else:
        bpp = 1 if mode == "8bit" else 4
        screen = torch.full((nframes, H, W * bpp), 0x5A, dtype=torch.uint8, device="cuda")
        fe.warp(d_faces, screen, nframes=nframes, rgba=mode != "8bit", tables=tables if mode == "tables" else None)
    torch.cuda.synchronize()
    return screen.cpu().numpy()


CASES = {
    "panini": ("cube", "panini", "f_fov 180", (640, 360, 256), False),
    "fisheye1": ("cube", "fisheye1", "f_contain", (640, 360, 256), False),
    "quincuncial": ("cube", "quincuncial", "f_cover", (640, 360, 256), True),
    "trism": ("trism", "panini", "f_fov 180", (480, 272, 192), False),
    "fast": ("fast", "panini", "f_fov 160", (480, 272, 192), True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_layout_warps_equal_the_dense_warp(bb, fe, torch_mod, restate, palette, case):
    torch = torch_mod
    globe, lens, zoom, size, rubix = CASES[case]
    setup(fe, globe, lens, zoom, size, rubix)
    W, H, ps, n = fe.width, fe.height, fe.platesize, fe.numplates
    bg = bb.synthetic_background(W, H)
    fe.set_background(bg)
    fe.set_rgba_table(np.random.default_rng(5).integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32))
    tables = torch.from_numpy(np.random.default_rng(6).integers(0, 2**31, (16, 256), dtype=np.int64).astype(np.int32)).cuda()
    faces = faces_batch(bb, fe, 16, 40)
    d_dense = torch.from_numpy(faces).cuda()
    idx, tint = fe.lensmap()
    want_oracle = restate.render(idx, tint, faces[0], restate.palmaps(palette), rubix, background=bg)
    for name, (rowbytes, origins, rows, kernel) in layouts(ps, n).items():
        surf = surfaces(faces, rowbytes, origins, rows, seed=len(name))
        d_surf = torch.from_numpy(surf).cuda()
        for nframes in (1, 5, 16):
            for mode in ("8bit", "rgba", "tables", "view-keep"):
                fe.set_face_layout()
                want = run(torch, fe, d_dense[:nframes], nframes, mode, tables)
                fe.set_face_layout(rowbytes, origins)
                got = run(torch, fe, d_surf[:nframes], nframes, mode, tables)
                k = fe.last_kernel
                assert np.array_equal(got, want), (case, name, nframes, mode, k, int((got != want).sum()))
                assert "layout=1" in k and kernel in k, (case, name, k)
                if mode == "8bit" and nframes == 1:
                    assert np.array_equal(got[0], want_oracle), (case, name)
        # gap independence: other bytes outside the plates, same output (BOX boxes that overhang a plate stage them)
        fe.set_face_layout(rowbytes, origins)
        want = run(torch, fe, d_surf, 16, "8bit")
        d_surf.copy_(torch.from_numpy(surfaces(faces, rowbytes, origins, rows, seed=99)))
        assert np.array_equal(run(torch, fe, d_surf, 16, "8bit"), want), (case, name)
        # the direct-gather kernel (blinky_set_kernel(1)) through the same layout
        fe.set_kernel(1)
        got = run(torch, fe, d_surf, 5, "rgba")
        assert "warp_gather_kernel" in fe.last_kernel and "layout=1" in fe.last_kernel, fe.last_kernel
        fe.set_kernel(0)
        fe.set_face_layout()
        assert np.array_equal(got, run(torch, fe, d_dense[:5], 5, "rgba")), (case, name)


def test_layout_per_pixel_kernel_for_an_odd_width(bb, fe, torch_mod):
    torch = torch_mod
    setup(fe, "cube", "quincuncial", "f_cover", (333, 201, 128), True)
    ps, n = fe.platesize, fe.numplates
    faces = faces_batch(bb, fe, 5, 7)
    d_dense = torch.from_numpy(faces).cuda()
    for name in ("atlas-3x2", "odd-origins"):
        rowbytes, origins, rows, _ = layouts(ps, n)[name]
        d_surf = torch.from_numpy(surfaces(faces, rowbytes, origins, rows, seed=3)).cuda()
        for nframes in (1, 5):
            for mode in ("8bit", "rgba"):
                fe.set_face_layout()
                want = run(torch, fe, d_dense[:nframes], nframes, mode)
                fe.set_face_layout(rowbytes, origins)
                got = run(torch, fe, d_surf[:nframes], nframes, mode)
                assert "warp_scalar_kernel" in fe.last_kernel and "layout=1" in fe.last_kernel, fe.last_kernel
                assert np.array_equal(got, want), (name, nframes, mode)


@pytest.mark.parametrize("keep", [False, True])
def test_warp_host_from_an_atlas(bb, fe, keep):
    setup(fe, "cube", "stereographic", "f_fov 200", (400, 240, 160), False)
    ps, n = fe.platesize, fe.numplates
    fe.set_background(bb.synthetic_background(fe.width, fe.height))
    faces = faces_batch(bb, fe, 4, 70)
    rowbytes, origins, rows, _ = layouts(ps, n)["odd-origins"]
    surf = surfaces(faces, rowbytes, origins, rows, seed=4)
    dst0 = np.random.default_rng(8).integers(0, 256, (4, fe.height + 4, fe.width + 10), dtype=np.uint8)
    want = fe.warp_host(faces.reshape(4, -1), dst0.copy(), keep_unmapped=keep, x0=6, y0=2)
    fe.set_face_layout(rowbytes, origins)
    got = fe.warp_host(surf, dst0.copy(), keep_unmapped=keep, x0=6, y0=2)
    assert np.array_equal(got, want), "pageable atlas"
    pinned = fe.alloc_pinned(surf.nbytes)
    try:
        pinned[:] = surf.reshape(-1)
        got = fe.warp_host(pinned, dst0.copy(), keep_unmapped=keep, x0=6, y0=2, nframes=4, face_stride=rows * rowbytes)
        assert np.array_equal(got, want), "pinned atlas"
    finally:
        fe.free_pinned(pinned)


def test_capture_keeps_the_layout_of_the_capture(bb, fe, torch_mod):
    torch = torch_mod
    setup(fe, "cube", "panini", "f_fov 180", (640, 360, 256), False)
    ps, n = fe.platesize, fe.numplates
    faces = faces_batch(bb, fe, 5, 90)
    rowbytes, origins, rows, _ = layouts(ps, n)["atlas-3x2"]
    d_surf = torch.from_numpy(surfaces(faces, rowbytes, origins, rows, seed=2)).cuda()
    out = torch.zeros((5, fe.height, fe.width), dtype=torch.uint8, device="cuda")
    fe.set_face_layout(rowbytes, origins)
    fe.warp(d_surf, out, nframes=5)
    torch.cuda.synchronize()
    want = out.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp(d_surf, out, nframes=5)
    assert "warp_ring_kernel" in fe.last_kernel and "layout=1" in fe.last_kernel, fe.last_kernel
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    # another layout (the plates stacked instead) set after the capture: the replay keeps reading the atlas
    fe.set_face_layout(ps, [(0, i * ps) for i in range(n)])
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    fe.set_face_layout()
    del g
    fe.release_captures()


def test_layout_that_no_longer_fits_is_refused(bb, fe, torch_mod):
    torch = torch_mod
    setup(fe, "cube", "panini", "f_fov 180", (320, 180, 128), False)
    rowbytes, origins, rows, _ = layouts(128, 6)["atlas-3x2"]
    d_surf = torch.zeros((2, rows, rowbytes), dtype=torch.uint8, device="cuda")
    fe.set_face_layout(rowbytes, origins)
    sentinel = torch.full((2, fe.height, fe.width), 0x5A, dtype=torch.uint8, device="cuda")
    out = sentinel.clone()
    fe.warp(d_surf, out, nframes=2)
    launches = fe.launch_count

    def refused(nframes=2, face_stride=None, **kw):
        out = torch.full((2, fe.height, fe.width * 4), 0x5A, dtype=torch.uint8, device="cuda")
        for rgba in (False, True):
            with pytest.raises(bb.BlinkyError) as e:
                fe.warp(d_surf, out, nframes=nframes, face_stride=face_stride, rgba=rgba)
            assert e.value.code == bb.E_INVALID, str(e.value)
        with pytest.raises(bb.BlinkyError) as e:
            fe.warp_view(d_surf, out, x0=0, y0=0, nframes=nframes, face_stride=face_stride, keep_unmapped=True)
        assert e.value.code == bb.E_INVALID
        torch.cuda.synchronize()
        assert bool((out == 0x5A).all()) and fe.launch_count == launches

    refused(face_stride=rows * rowbytes - 1)          # frames overlap
    fe.build_lensmap(320, 180, 256, 8)                 # a larger plate size: the plates overhang rowbytes
    refused()
    fe.set_face_layout(rowbytes, origins[:2])          # two origins...
    fe.command("f_globe fast")
    fe.build_lensmap(320, 180, 128, 8)
    fe.warp(d_surf, out, nframes=2)                    # ...are enough for fast
    launches = fe.launch_count
    fe.command("f_globe cube")                         # ...but not for cube
    fe.build_lensmap(320, 180, 128, 8)
    refused()
    # a fast-style globe whose globe_plate also returns plate 2, a slot the cube left behind
    src = open(os.path.join(bb.SCRIPT_DIR, "lua-scripts", "globes", "fast.lua")).read()
    assert "  return BIG\n" in src
    fe.load_globe("stale", src.replace("  return BIG\n", "  if x > 0.3 then return 2 end\n  return BIG\n"))
    fe.build_lensmap(320, 180, 128, 8)
    assert fe.numplates == 2
    refused()
    fe.set_face_layout(rowbytes, origins[:3])
    fe.warp(d_surf, out, nframes=2)
    torch.cuda.synchronize()


def test_full_size_atlas(bb, fe, torch_mod):
    """4K, 6 x 2048^2 plates in a 3x2 atlas, 16 frames"""
    torch = torch_mod
    setup(fe, "cube", "panini", "f_fov 180", (3840, 2160, 2048), False)
    ps, n = fe.platesize, fe.numplates
    rowbytes, origins, rows, _ = layouts(ps, n)["atlas-3x2"]
    gen = torch.Generator(device="cuda").manual_seed(1)
    d_dense = torch.randint(0, 256, (16, n, ps, ps), dtype=torch.uint8, device="cuda", generator=gen)
    d_surf = torch.randint(0, 256, (16, rows, rowbytes), dtype=torch.uint8, device="cuda", generator=gen)
    for i, (x, y) in enumerate(origins):
        d_surf[:, y:y + ps, x:x + ps] = d_dense[:, i]
    for mode in ("8bit", "rgba"):
        want = run(torch, fe, d_dense, 16, mode)
        fe.set_face_layout(rowbytes, origins)
        got = run(torch, fe, d_surf, 16, mode)
        assert "warp_ring_kernel" in fe.last_kernel and "layout=1" in fe.last_kernel, fe.last_kernel
        fe.set_face_layout()
        assert np.array_equal(got, want), mode
