"""The device-resident warp into a view rectangle of a pitched device framebuffer (blinky_warp_device_view and
its RGBA form), on the GPU.

Checked against the compiled reference's golden frames (rendered into a view rectangle of a larger screen,
unmapped pixels left alone) and against the CPU oracle, for views the fast kernels take (origin, pitch and
frame stride multiples of 4 pixels) and views they cannot (the per-pixel kernel).  Every byte of the screen
outside the rectangle, and with keep_unmapped every unmapped pixel inside it, must keep the caller's fill."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch

    return torch


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


def setup(fe, globe, lens, w, h, ps, zoom=None, rubix=False):
    fe.command(f"f_globe {globe}")
    fe.command(f"f_lens {lens}")
    if zoom:
        fe.command(zoom)
    fe.set_rubix(rubix)
    fe.build_lensmap(w, h, ps, 8)


def rgba_table():
    return np.random.default_rng(5).integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32)


def stream_of(torch):
    return torch.cuda.current_stream().cuda_stream


def warp_into_screen(torch, fe, d_faces, want8, mapped, *, nframes, x0, y0, rowbytes, rows_below, pad, keep, rgba,
                     table=None, seed=0):
    """Warps `nframes` frames into a random-filled flat device buffer of screens (rows_below guard rows under the
    rectangle, `pad` bytes between screens) and checks every byte of it.  Returns the kernel that ran."""
    W, H = fe.width, fe.height
    bpp = 4 if rgba else 1
    fstride = (y0 + H + rows_below) * rowbytes + pad
    fill = np.random.default_rng(seed).integers(0, 256, nframes * fstride, dtype=np.uint8)
    d_screen = torch.from_numpy(fill).cuda()
    fe.warp_view(d_faces, d_screen.data_ptr(), x0=x0, y0=y0, rowbytes=rowbytes, nframes=nframes, keep_unmapped=keep,
                 rgba=rgba, screen_stride=fstride, stream=stream_of(torch))
    torch.cuda.synchronize()
    got = d_screen.cpu().numpy()
    expect = fill.copy()
    mask = np.repeat(mapped, bpp, axis=1)
    for f in range(nframes):
        start = f * fstride + y0 * rowbytes
        rect = expect[start:start + H * rowbytes].reshape(H, rowbytes)[:, x0 * bpp:(x0 + W) * bpp]
        px = table[want8[f]].view(np.uint8).reshape(H, W * 4) if rgba else want8[f]
        if keep:
            rect[mask] = px[mask]
        else:
            rect[:] = px
    assert np.array_equal(got, expect), (fe.last_kernel, nframes, x0, y0, rowbytes, keep, rgba)
    return fe.last_kernel


# ---- golden frames of the compiled reference, device path -------------------------------------------------------

@pytest.mark.parametrize("kernel", [0, 1])
def test_golden_frames_device_view(bb, fe, torch_mod, kernel):
    """frames_small.npz were rendered by the compiled reference into a 160x120 screen with scr_vrect = (8, 6, 128, 96)
    and unmapped pixels left alone: the device view with keep_unmapped reproduces them byte for byte, and the RGBA
    form gives the same frames through the palette table"""
    torch = torch_mod
    frames = np.load(os.path.join(G, "frames_small.npz"))
    W, H, PS = 128, 96, 48
    table = rgba_table()
    fe.set_rgba_table(table)
    for key in frames.files:
        g, l, r = key.split("__")
        setup(fe, g, l, W, H, PS, None, r == "rubix1")
        fe.set_kernel(kernel)
        faces = torch.from_numpy(bb.synthetic_faces(fe.numplates, PS, 0)).cuda()
        screen = np.random.default_rng(3).integers(0, 256, (120, 160), dtype=np.uint8)  # what Draw_TileClear left
        d_screen = torch.from_numpy(screen.reshape(1, 120, 160)).cuda()
        fe.warp_view(faces, d_screen, x0=8, y0=6, keep_unmapped=True, stream=stream_of(torch))
        d_rgba = torch.from_numpy(table[screen].view(np.int32).reshape(1, 120, 160)).cuda()
        fe.warp_view(faces, d_rgba, x0=8, y0=6, keep_unmapped=True, rgba=True, stream=stream_of(torch))
        torch.cuda.synchronize()
        # (kernel 0: plans without BOX tiles run in the GATHER-tile kernel alone)
        tiled = "warp_ring_kernel" in fe.last_kernel or "warp_tile_gather_kernel" in fe.last_kernel
        assert (tiled if kernel == 0 else "warp_gather_kernel" in fe.last_kernel), (key, fe.last_kernel)
        assert np.array_equal(d_screen.cpu().numpy()[0], frames[key]), (key, kernel)
        assert np.array_equal(d_rgba.cpu().numpy()[0].view(np.uint32), table[frames[key]]), (key, kernel)


# ---- oracle sweep ------------------------------------------------------------------------------------------------

SWEEP = {
    "panini-rubix": ("cube", "panini", None, (320, 200, 128), True),
    "hammer-contain-rubix": ("tetra", "hammer", "f_contain", (400, 226, 192), True),   # BOX, GATHER and EMPTY tiles
    "quincuncial-cover": ("cube", "quincuncial", "f_cover", (320, 200, 256), False),   # large boxes
    "fisheye1-ragged": ("cube", "fisheye1", None, (322, 150, 96), True),               # W % 4 != 0
}


def views(W, bpp):
    """(name, x0, y0, rowbytes, pad): an aligned view, an origin that is not 4-aligned, a pitch that is not 4 pixels"""
    aligned = -(-(8 + W + 13) * bpp // 16) * 16
    return [("aligned", 8, 2, aligned, 64),
            ("odd-origin", 3, 1, aligned, 7 * bpp),
            ("odd-pitch", 8, 2, (8 + W + 3) * bpp, 7 * bpp)]


@pytest.mark.parametrize("case", list(SWEEP))
def test_view_against_oracle(bb, fe, restate, palette, torch_mod, case):
    torch = torch_mod
    globe, lens, zoom, (W, H, PS), rubix = SWEEP[case]
    setup(fe, globe, lens, W, H, PS, zoom, rubix)
    bg = bb.synthetic_background(W, H)
    fe.set_background(bg)
    table = rgba_table()
    fe.set_rgba_table(table)
    if case.startswith("hammer"):
        types = set(fe.tile_plan()[0]["type"] & 3)
        assert {0, 2} <= types and types & {1, 3}, types   # EMPTY, GATHER and BOX tiles
    idx, tint = fe.lensmap()
    mapped = idx >= 0
    pm = restate.palmaps(palette)
    faces = np.stack([bb.synthetic_faces(fe.numplates, PS, 50 + i) for i in range(16)])
    want8 = np.stack([restate.render(idx, tint, faces[i], pm, rubix, background=bg) for i in range(16)])
    d_faces = torch.from_numpy(faces).cuda()
    seed = 0
    for nframes in (1, 5, 16):
        for rgba in (False, True):
            for name, x0, y0, rowbytes, pad in views(W, 4 if rgba else 1):
                for keep in (False, True):
                    seed += 1
                    kernel = warp_into_screen(torch, fe, d_faces, want8, mapped, nframes=nframes, x0=x0, y0=y0,
                                              rowbytes=rowbytes, rows_below=3, pad=pad, keep=keep, rgba=rgba,
                                              table=table, seed=seed)
                    fast = name == "aligned" and W % 4 == 0
                    assert ("warp_ring_kernel" if fast else "warp_scalar_kernel") in kernel, (case, name, kernel)
                    assert ("keep=1" in kernel) == keep, kernel


# ---- ring geometries with keep_unmapped -------------------------------------------------------------------------

KEEP_RING_KNOBS = [
    {"BLINKY_RING_BYTES": "128", "BLINKY_RING_BOXES": "6"},  # the smallest ring the plan allows: wraps all the time
    {"BLINKY_RING_CTAS": "2", "BLINKY_STATIC_PCT": "0"},     # every unit from the ticket counter
    {"BLINKY_RING_CTAS": "16", "BLINKY_STATIC_PCT": "100"},  # no tickets
    {"BLINKY_FCHUNK": "1"}, {"BLINKY_FCHUNK": "3"}, {"BLINKY_FCHUNK": "16"},
]


@pytest.mark.parametrize("knobs", KEEP_RING_KNOBS, ids=lambda k: ",".join(f"{a[7:]}={b}" for a, b in k.items()))
def test_keep_unmapped_ring_geometries(bb, restate, palette, torch_mod, cuda_device, knobs, monkeypatch):
    """With keep_unmapped the ring kernel's units are the BOX tiles alone; its schedules and ring geometries still
    never change the pixels.  Launches of 5 frames (GATHER tiles ride in the ring kernel's launch) and 16 (in front
    of it), one after the other on one stream, so the ticket bookkeeping of the smaller unit count is exercised."""
    torch = torch_mod
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    globe, lens, zoom, (W, H, PS), rubix = SWEEP["hammer-contain-rubix"]
    with bb.Fisheye(device=cuda_device, palette=palette) as f:   # the knobs are read when the context is created
        setup(f, globe, lens, W, H, PS, zoom, rubix)
        f.set_background(bb.synthetic_background(W, H))
        table = rgba_table()
        f.set_rgba_table(table)
        idx, tint = f.lensmap()
        pm = restate.palmaps(palette)
        faces = np.stack([bb.synthetic_faces(f.numplates, PS, 70 + i) for i in range(16)])
        want8 = np.stack([restate.render(idx, tint, faces[i], pm, rubix) for i in range(16)])
        d_faces = torch.from_numpy(faces).cuda()
        for nframes in (5, 16, 5):
            for rgba in (False, True):
                bpp = 4 if rgba else 1
                kernel = warp_into_screen(torch, f, d_faces, want8, idx >= 0, nframes=nframes, x0=4, y0=3,
                                          rowbytes=(W + 16) * bpp, rows_below=2, pad=16 * bpp, keep=True, rgba=rgba,
                                          table=table, seed=nframes + bpp)
                assert "warp_ring_kernel" in kernel and "keep=1" in kernel, kernel


# ---- the dense form is the view that is the whole screen ----------------------------------------------------------

def test_dense_view_is_warp(bb, fe, torch_mod):
    torch = torch_mod
    W, H, PS, N = 320, 200, 128, 3
    setup(fe, "tetra", "hammer", W, H, PS, "f_contain", True)
    fe.set_background(bb.synthetic_background(W, H))
    fe.set_rgba_table(rgba_table())
    d_faces = torch.from_numpy(np.stack([bb.synthetic_faces(fe.numplates, PS, i) for i in range(N)])).cuda()
    for kernel in (0, 1):
        fe.set_kernel(kernel)
        for rgba, dtype in ((False, torch.uint8), (True, torch.int32)):
            a = torch.zeros((N, H, W), dtype=dtype, device="cuda")
            b = torch.full((N, H, W), 7, dtype=dtype, device="cuda")
            fe.warp(d_faces, a, nframes=N, rgba=rgba, stream=stream_of(torch))
            fe.warp_view(d_faces, b, rowbytes=W * (4 if rgba else 1), x0=0, y0=0, nframes=N, keep_unmapped=False,
                         rgba=rgba, stream=stream_of(torch))
            torch.cuda.synchronize()
            assert torch.equal(a, b), (kernel, rgba)


# ---- split screen: two contexts, one screen ------------------------------------------------------------------------

@pytest.mark.parametrize("rgba", [False, True])
def test_split_screen_two_contexts(bb, restate, palette, torch_mod, cuda_device, rgba):
    """Two contexts with different lenses write adjoining rectangles of one screen with keep_unmapped, on one stream;
    the seam is at x0 = 162, not a multiple of 4.  Each rectangle matches its oracle, the rest keeps its fill."""
    torch = torch_mod
    H, PS, N = 120, 96, 2
    left = ("cube", "panini", None, 160, False)
    right = ("tetra", "hammer", "f_contain", 148, True)
    x0s = (2, 2 + left[3])
    SW, SH, y0 = 2 + left[3] + right[3] + 6, H + 10, 4
    bpp = 4 if rgba else 1
    table = rgba_table()
    fill = np.random.default_rng(11).integers(0, 256, (N, SH, SW * bpp), dtype=np.uint8)
    d_screen = torch.from_numpy(fill).cuda()
    expect = fill.copy()
    pm = restate.palmaps(palette)
    ctxs, d_faces = [], []
    try:
        for (globe, lens, zoom, W, rubix), x0 in zip((left, right), x0s):
            f = bb.Fisheye(device=cuda_device, palette=palette)
            ctxs.append(f)
            setup(f, globe, lens, W, H, PS, zoom, rubix)
            f.set_rgba_table(table)
            idx, tint = f.lensmap()
            faces = np.stack([bb.synthetic_faces(f.numplates, PS, 90 + i) for i in range(N)])
            d_faces.append(torch.from_numpy(faces).cuda())
            f.warp_view(d_faces[-1], d_screen, x0=x0, y0=y0, rowbytes=SW * bpp, nframes=N,
                        keep_unmapped=True, rgba=rgba, screen_stride=SH * SW * bpp, stream=stream_of(torch))
            mask = np.repeat(idx >= 0, bpp, axis=1)
            for i in range(N):
                want = restate.render(idx, tint, faces[i], pm, rubix)
                px = table[want].view(np.uint8).reshape(H, W * 4) if rgba else want
                rect = expect[i, y0:y0 + H, x0 * bpp:(x0 + W) * bpp]
                rect[mask] = px[mask]
        torch.cuda.synchronize()
        assert np.array_equal(d_screen.cpu().numpy(), expect)
    finally:
        for f in ctxs:
            f.close()


# ---- argument errors --------------------------------------------------------------------------------------------

def test_view_argument_errors_launch_nothing(bb, fe, torch_mod):
    torch = torch_mod
    W, H, PS = 128, 96, 48
    setup(fe, "cube", "panini", W, H, PS)
    d_faces = torch.from_numpy(np.stack([bb.synthetic_faces(6, PS, i) for i in range(2)])).cuda()
    screen = torch.zeros(4 * 200 * 160 * 4 + 64, dtype=torch.uint8, device="cuda")
    base = screen.data_ptr()
    ok = dict(x0=8, y0=6, rowbytes=160, nframes=2, screen_stride=120 * 160)
    ok4 = dict(x0=8, y0=6, rowbytes=640, nframes=2, screen_stride=120 * 640, rgba=True)
    bad = [
        ("NULL faces", None, base, ok),
        ("NULL screen", d_faces, None, ok),
        ("x0 < 0", d_faces, base, {**ok, "x0": -1}),
        ("y0 < 0", d_faces, base, {**ok, "y0": -1}),
        ("rowbytes", d_faces, base, {**ok, "rowbytes": 8 + W - 1}),
        ("rowbytes RGBA", d_faces, base, {**ok4, "rowbytes": (8 + W) * 4 - 4}),
        ("frame stride", d_faces, base, {**ok, "screen_stride": (6 + H) * 160 - 1}),
        ("RGBA origin", d_faces, base + 1, ok4),
        ("RGBA pitch", d_faces, base, {**ok4, "rowbytes": 642}),
        ("RGBA stride", d_faces, base, {**ok4, "screen_stride": 120 * 640 + 2}),
    ]
    before = fe.launch_count
    for name, faces, scr, kw in bad:
        with pytest.raises(bb.BlinkyError) as e:
            fe.warp_view(0 if faces is None else faces, 0 if scr is None else scr, **kw)
        assert e.value.code == bb.E_INVALID, name
        assert fe.launch_count == before, name
    # the same arguments made valid do launch
    fe.warp_view(d_faces, base, **ok)
    fe.warp_view(d_faces, base, **ok4)
    torch.cuda.synchronize()
    assert fe.launch_count > before


def test_dense_null_buffers_and_negative_host_origin_launch_nothing(bb, fe, torch_mod):
    """the dense entry points refuse a NULL buffer as the view entry points do, and blinky_warp_host a negative view
    origin: nothing is launched and nothing is written"""
    torch = torch_mod
    W, H, PS = 128, 96, 48
    setup(fe, "cube", "panini", W, H, PS)
    lib = bb.load_library()
    faces = np.stack([bb.synthetic_faces(6, PS, i) for i in range(2)])
    d_faces = torch.from_numpy(faces).cuda()
    out = torch.full((2 * W * H * 4,), 0xA5, dtype=torch.uint8, device="cuda")
    before = fe.launch_count
    for fn, name, bpp in ((lib.blinky_warp_device, "blinky_warp_device", 1), (lib.blinky_warp_device_rgba, "blinky_warp_device_rgba", 4)):
        for f, o in ((None, out.data_ptr()), (d_faces.data_ptr(), None)):
            assert fn(fe._ctx, f, faces[0].nbytes, o, bpp * W * H, 2, None) == bb.E_INVALID
            assert lib.blinky_last_error(fe._ctx).decode() == f"{name}: NULL buffer"
    torch.cuda.synchronize()
    assert bool((out == 0xA5).all())
    rowbytes, guard = W + 16, 4096
    dst = np.full(guard + 2 * (H + 8) * rowbytes + guard, 0xA5, np.uint8)
    for x0, y0 in ((-1, 0), (0, -1), (-1, -1)):
        rc = lib.blinky_warp_host(fe._ctx, faces.ctypes.data, faces[0].nbytes, dst.ctypes.data + guard, (H + 8) * rowbytes, rowbytes, x0, y0, 2, 0)
        assert rc == bb.E_INVALID, (x0, y0)
        assert lib.blinky_last_error(fe._ctx).decode() == "the view origin (x0, y0) must not be negative"
    assert (dst == 0xA5).all()
    assert fe.launch_count == before
