"""The warps and the device lensmap build at the limits of their index ranges, on the GPU.

Each case stays near one narrow field or hard limit of the kernels: screens past the 16-bit tile origins, plates at
the 28-bit texel index, batches and face surfaces past 2^32 bytes, the 64 MB output pitch, the 65535-frame grid and
the forward builder's cap on undecided grid points.  Every warp is compared with torch's own gather of the
context's lensmap (out = where(valid, lut[tint][faces[idx]], background), then the RGBA table), and the lensmaps
with the oracle's C transcription or the interpreter.  Each case runs through every kernel that can take it: the
default choice (the ring kernel where there is a tile plan), K1 (set_kernel(1)), K0 (a view at an odd x0) and K3
(BLINKY_SERIAL_GATHER=1: GATHER tiles in their own kernel); `last_kernel` shows which one ran.

The large cases allocate up to about 7 GB of device memory and free it before the next case."""
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
KERNEL = {"ring": "warp_ring_kernel", "K1": "warp_gather_kernel", "K0": "warp_scalar_kernel", "K3": "warp_tile_gather_kernel"}
MAX_PS = 6688


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch

    return torch


@pytest.fixture(autouse=True)
def _free_device_memory(torch_mod):
    yield
    gc.collect()
    torch_mod.cuda.empty_cache()


@pytest.fixture()
def ctxs(bb, palette, cuda_device, monkeypatch):
    """(a context with the default kernel choice, one that launches GATHER tiles in their own kernel K3)"""
    fe = bb.Fisheye(device=cuda_device, palette=palette)
    monkeypatch.setenv("BLINKY_SERIAL_GATHER", "1")
    fe3 = bb.Fisheye(device=cuda_device, palette=palette)
    monkeypatch.delenv("BLINKY_SERIAL_GATHER")
    yield fe, fe3
    fe.close()
    fe3.close()


def setup(fes, globe, lens, zoom, size, rubix, threads=0, lens_source=None):
    W, H, PS = size
    for fe in fes:
        fe.command(f"f_globe {globe}")
        if lens_source:
            fe.load_lens(lens, lens_source)
        else:
            fe.command(f"f_lens {lens}")
            fe.command(zoom)
        fe.set_rubix(rubix)
        fe.build_lensmap(W, H, PS, threads=threads)


def oracle_map(fe, restate, globe, lens, zoom):
    z = zoom.split()
    om = restate.build(globe, lens, fe.width, fe.height, fe.platesize, zoom=(z[0], int(z[1]) if len(z) > 1 else 0))
    idx, tint = fe.lensmap()
    assert np.array_equal(idx, om["idx"]) and np.array_equal(tint, om["tint"]), fe.build_info
    return om


class Reference:
    """torch's own gather of a context's lensmap"""

    def __init__(self, torch, fe, bg, table=None):
        self.torch = torch
        idx, tint = fe.lensmap()
        self.H, self.W = idx.shape
        i = torch.from_numpy(idx.reshape(-1).astype(np.int64)).cuda()
        self.valid = i >= 0
        self.idx = i.clamp(min=0)
        self.tint = torch.from_numpy(np.where(tint == 255, 6, tint).reshape(-1).astype(np.int64)).cuda()
        self.lut = torch.from_numpy(np.concatenate([fe.palmaps(), np.arange(256, dtype=np.uint8)[None]])).cuda()
        self.rubix = fe.rubix_enabled
        self.bg = torch.from_numpy(np.ascontiguousarray(bg).reshape(-1)).cuda()
        self.table = None if table is None else torch.from_numpy(table.view(np.int32)).cuda()

    def frames(self, faces2d):
        """faces2d: [n, texels] (any strides) -> [n, H, W], uint8 or (with a table) int32"""
        src = faces2d[:, self.idx]
        if self.rubix:
            src = self.lut[self.tint, src.long()]
        out = self.torch.where(self.valid, src, self.bg)
        if self.table is not None:
            out = self.table[out.long()]
        return out.reshape(-1, self.H, self.W)

    def check(self, faces2d, got, what):
        """every frame of `got` ([n, H, W]) against frames(faces2d), a few frames at a time"""
        chunk, n = max(1, (1 << 25) // (self.H * self.W)), got.shape[0]
        for f0 in range(0, n, chunk):
            want = self.frames(faces2d[f0:min(f0 + chunk, n)])
            ok = got[f0:f0 + chunk] == want
            if not bool(ok.all()):
                bad = (~ok).reshape(ok.shape[0], -1)
                f = f0 + int(bad.any(1).nonzero()[0])
                raise AssertionError(f"{what}: frame {f} differs in {int(bad[f - f0].sum())} pixels")


def warp(torch, fe, how, d_faces, nframes, rgba=False, face_stride=None):
    """one warp into sentinel-filled frames through `how` ("ring": the context's own choice, "K1", "K0": the view at
    x0 = 1 of screens one pixel wider); returns ([nframes, H, W] uint8 or int32, last_kernel)"""
    W, H, bpp = fe.width, fe.height, 4 if rgba else 1
    fe.set_kernel(1 if how == "K1" else 0)
    try:
        if how == "K0":
            screen = torch.full((nframes, H, (W + 1) * bpp), SENTINEL, dtype=torch.uint8, device="cuda")
            fe.warp_view(d_faces, screen, x0=1, nframes=nframes, rgba=rgba, face_stride=face_stride)
            out = screen.view(torch.int32)[:, :, 1:] if rgba else screen[:, :, 1:]
        else:
            screen = torch.full((nframes, H, W * bpp), SENTINEL, dtype=torch.uint8, device="cuda")
            fe.warp(d_faces, screen, nframes=nframes, face_stride=face_stride, rgba=rgba)
            out = screen.view(torch.int32) if rgba else screen
    finally:
        fe.set_kernel(0)
    torch.cuda.synchronize()
    return out, fe.last_kernel


def rgba_table(seed=5):
    return np.random.default_rng(seed).integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32)


def has_gather_tiles(fe):
    tiles, _ = fe.tile_plan()
    return bool(((tiles["type"] & 3) == 2).any())


def tiled_runs(fe, fe3):
    """(context, how, kernel that must run) for the default choice, K1, K0 and K3.  The default choice is the ring
    kernel, with K3 alone for a plan of nothing but GATHER tiles; the serial-gather context adds K3 when the default
    does not run it anyway."""
    types = fe.tile_plan()[0]["type"] & 3
    only_gather = bool((types == 2).all())
    runs = [(fe, "ring", KERNEL["K3"] if only_gather else KERNEL["ring"]), (fe, "K1", KERNEL["K1"]), (fe, "K0", KERNEL["K0"])]
    if (types == 2).any() and not only_gather:
        runs.append((fe3, "ring", KERNEL["K3"]))
    return runs


# -- 1. screens wider or taller than 65536 pixels ---------------------------------------------------------------


@pytest.mark.parametrize("W,H", [(65600, 64), (64, 65600), (65536, 64), (64, 65536)])
def test_screens_past_the_16_bit_tile_origins(bb, ctxs, torch_mod, restate, W, H):
    """A tile plan holds 16-bit tile origins: up to 65536 pixels the ring kernel warps the screen, past that the flat
    kernels do, and every pixel is right.  The lens kernel's grid has one row per screen row, so screens taller than
    65535 rows are built by the interpreter, with that reason in build_info."""
    torch = torch_mod
    fe, fe3 = ctxs
    ps = 16
    setup((fe, fe3), "cube", "equirect", "f_cover", (W, H, ps), True)
    oracle_map(fe, restate, "cube", "equirect", "f_cover")
    oracle_map(fe3, restate, "cube", "equirect", "f_cover")
    if H > 65535:
        assert fe.build_info.startswith("host (screen taller than 65535 rows"), fe.build_info
    else:
        assert fe.build_info.startswith("device"), fe.build_info
    planned = max(W, H) <= 65536
    tiles, _ = fe.tile_plan()
    assert (tiles.size > 0) == planned
    bg = bb.synthetic_background(W, H)
    table = rgba_table()
    for f in (fe, fe3):
        f.set_background(bg)
        f.set_rgba_table(table)
    n = 2
    d_faces = torch.randint(0, 256, (n, 6 * ps * ps), dtype=torch.uint8, device="cuda",
                            generator=torch.Generator(device="cuda").manual_seed(W + H))
    for rgba in (False, True):
        ref = Reference(torch, fe, bg, table if rgba else None)
        runs = tiled_runs(fe, fe3) if planned else [(fe, "ring", KERNEL["K1"]), (fe, "K1", KERNEL["K1"]), (fe, "K0", KERNEL["K0"])]
        for ctx, how, kernel in runs:
            got, k = warp(torch, ctx, how, d_faces, n, rgba)
            assert kernel in k, (W, H, how, k)
            ref.check(d_faces, got, f"{W}x{H} rgba={rgba} {how}: {k}")
            del got


# -- 2. plates at the 28-bit texel index limit ------------------------------------------------------------------

# a narrow view into the far corner of the cube's bottom plate (5), magnified: BOX tiles whose boxes TMA stages from
# more than 6000 texels into a 6688 plate, at plate coordinate 5
CORNER_ZOOM_LENS = """lens_width=0.1 lens_height=0.05625 onload='f_contain'
function lens_inverse(x, y) return 0.9 + x, -1, -0.9 + y end"""


@pytest.mark.parametrize("lens,rubix", [("panini", False), ("panini", True), ("corner_zoom", True)])
def test_plates_at_the_texel_index_limit(bb, ctxs, torch_mod, restate, palette, lens, rubix):
    """Cube of 6688^2 plates (44.7 MB each) at 1920x1080: panini f_fov 180 samples every plate through GATHER tiles;
    the corner view is all BOX tiles deep in plate 5.  Three frames (0.8 GB of faces), dense and from a 3x2 atlas."""
    torch = torch_mod
    fe, fe3 = ctxs
    W, H, ps = 1920, 1080, MAX_PS
    setup((fe, fe3), "cube", lens, "f_fov 180", (W, H, ps), rubix, lens_source=CORNER_ZOOM_LENS if lens == "corner_zoom" else None)
    assert fe.build_info.startswith("device"), fe.build_info
    idx, tint = fe.lensmap()
    if lens == "panini":
        om = oracle_map(fe, restate, "cube", "panini", "f_fov 180")
        assert int(idx.max()) >= 4 * ps * ps   # the top or bottom plate is sampled
    else:
        # no C transcription of this lens: the interpreter's map is the reference
        with bb.Fisheye(device=None, palette=palette) as host:
            setup((host,), "cube", lens, None, (W, H, ps), rubix, threads=bb.usable_cpus(), lens_source=CORNER_ZOOM_LENS)
            hidx, htint = host.lensmap()
        assert np.array_equal(idx, hidx) and np.array_equal(tint, htint)
        assert int(idx[idx >= 0].min()) >= 5 * ps * ps
        tiles, _ = fe.tile_plan()
        assert ((tiles["type"] & 3) != 2).all() and int(tiles["box_y"].min()) > 6000
    bg = bb.synthetic_background(W, H)
    for f in (fe, fe3):
        f.set_background(bg)
    n = 3
    d_faces = torch.randint(0, 256, (n, 6, ps, ps), dtype=torch.uint8, device="cuda",
                            generator=torch.Generator(device="cuda").manual_seed(66))
    faces2d = d_faces.reshape(n, -1)
    ref = Reference(torch, fe, bg)
    runs = tiled_runs(fe, fe3)
    dense = None
    for ctx, how, kernel in runs:
        got, k = warp(torch, ctx, how, d_faces, n)
        assert kernel in k, (lens, how, k)
        ref.check(faces2d, got, f"ps {ps} {lens} {how}: {k}")
        if dense is None:
            dense = got
    if lens == "panini":
        want = restate.render(om["idx"], om["tint"], d_faces[0].cpu().numpy(), restate.palmaps(palette), rubix, background=bg)
        assert np.array_equal(dense[0].cpu().numpy(), want)

    # the same frames from a 3x2 atlas: rowbytes 3 * 6688 = 20064, a multiple of 16, so BOX tiles still go through TMA
    rowbytes, rows = 3 * ps, 2 * ps
    origins = [(c * ps, r * ps) for r in range(2) for c in range(3)]
    surf = torch.full((n, rows, rowbytes), SENTINEL, dtype=torch.uint8, device="cuda")
    for i, (x, y) in enumerate(origins):
        surf[:, y:y + ps, x:x + ps] = d_faces[:, i]
    for ctx, how, kernel in runs:
        ctx.set_face_layout(rowbytes, origins)
        try:
            got, k = warp(torch, ctx, how, surf, n)
        finally:
            ctx.set_face_layout()
        assert kernel in k and "layout=1" in k, (lens, how, k)
        assert torch.equal(got, dense), (lens, how, k)


# -- 3. batches past 4 GiB --------------------------------------------------------------------------------------


def test_faces_batch_past_4_gib(bb, ctxs, torch_mod):
    """175 frames of 6x2048^2 faces, 1552 bytes of padding between frames (a stride that is no power of two):
    4.4 GB of faces, so the later frames lie past 2^32 bytes.  Every frame is checked, the one that straddles
    2^32 included."""
    torch = torch_mod
    fe, fe3 = ctxs
    W, H, ps = 3840, 2160, 2048
    setup((fe, fe3), "cube", "panini", "f_fov 180", (W, H, ps), False)
    texels = 6 * ps * ps
    stride = texels + 1552
    n = 175
    assert (n - 1) * stride > 1 << 32 and (1 << 32) // stride < n - 1
    straddle = (1 << 32) // stride
    assert straddle * stride < 1 << 32 < straddle * stride + texels
    bg = bb.synthetic_background(W, H)
    for f in (fe, fe3):
        f.set_background(bg)
    buf = torch.randint(0, 256, (n * stride,), dtype=torch.uint8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    faces2d = buf.as_strided((n, texels), (stride, 1))
    ref = Reference(torch, fe, bg)
    assert has_gather_tiles(fe)
    for ctx, how, kernel in tiled_runs(fe, fe3):
        got, k = warp(torch, ctx, how, buf, n, face_stride=stride)
        assert kernel in k, (how, k)
        ref.check(faces2d, got, f"{n} frames, stride {stride}, {how}: {k}")
        del got


def test_rgba_output_past_4_gib(bb, ctxs, torch_mod):
    """132 RGBA frames at 3840x2160 (33.2 MB each): 4.4 GB of output, so frame 129 straddles 2^32 bytes and the
    frames after it are written past it.  Every frame is checked."""
    torch = torch_mod
    fe, fe3 = ctxs
    W, H, ps = 3840, 2160, 1024
    setup((fe, fe3), "cube", "panini", "f_fov 180", (W, H, ps), True)
    n = 132
    frame = W * H * 4
    assert 129 * frame < 1 << 32 < 130 * frame
    bg = bb.synthetic_background(W, H)
    table = rgba_table(9)
    for f in (fe, fe3):
        f.set_background(bg)
        f.set_rgba_table(table)
    d_faces = torch.randint(0, 256, (n, 6 * ps * ps), dtype=torch.uint8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    ref = Reference(torch, fe, bg, table)
    assert has_gather_tiles(fe)
    for ctx, how, kernel in tiled_runs(fe, fe3):
        got, k = warp(torch, ctx, how, d_faces, n, rgba=True)
        assert kernel in k, (how, k)
        ref.check(d_faces, got, f"{n} RGBA frames, {how}: {k}")
        del got


# -- 4. a face-layout surface larger than 4 GiB -----------------------------------------------------------------


def test_face_layout_surface_past_4_gib(bb, ctxs, torch_mod):
    """One frame: six 2048^2 plates stacked vertically in a surface with rows of 2^19 bytes, each at its own x
    (multiples of 16, so BOX tiles use TMA): 6.4 GB, and the plates 4 and 5 start at and past 2^32 bytes."""
    torch = torch_mod
    fe, fe3 = ctxs
    W, H, ps = 3840, 2160, 2048
    setup((fe, fe3), "cube", "panini", "f_fov 180", (W, H, ps), True)
    rowbytes = 1 << 19
    origins = [(16 * (1 + 997 * i) % (rowbytes - ps), i * ps) for i in range(6)]
    bases = [y * rowbytes + x for x, y in origins]
    assert bases[4] >= 1 << 32 and bases[5] > 1 << 32
    bg = bb.synthetic_background(W, H)
    for f in (fe, fe3):
        f.set_background(bg)
    d_faces = torch.randint(0, 256, (1, 6, ps, ps), dtype=torch.uint8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    surf = torch.full((6 * ps, rowbytes), SENTINEL, dtype=torch.uint8, device="cuda")
    for i, (x, y) in enumerate(origins):
        surf[y:y + ps, x:x + ps] = d_faces[0, i]
    ref = Reference(torch, fe, bg)
    assert has_gather_tiles(fe)
    for ctx, how, kernel in tiled_runs(fe, fe3):
        ctx.set_face_layout(rowbytes, origins)
        try:
            got, k = warp(torch, ctx, how, surf, 1, face_stride=6 * ps * rowbytes)
        finally:
            ctx.set_face_layout()
        assert kernel in k and "layout=1" in k, (how, k)
        ref.check(d_faces.reshape(1, -1), got, f"6.4 GB surface, {how}: {k}")


# -- 5. output pitch at the 64 MB limit -------------------------------------------------------------------------


@pytest.mark.parametrize("rgba", [False, True])
def test_output_pitch_at_64_mb(bb, ctxs, torch_mod, rgba):
    """A 256x64 view at (x0, 3) of a screen whose rows are 2^26 bytes apart, the largest pitch the warps take (four
    rows are 2^28 bytes: the ring kernel's 32-bit row step).  Fisheye f_contain leaves pixels unmapped, so the plan
    has BOX, GATHER and EMPTY tiles.  Only the view rectangle may change; a pitch 16 bytes larger is refused."""
    torch = torch_mod
    fe, fe3 = ctxs
    W, H, ps = 256, 64, 128
    setup((fe, fe3), "cube", "fisheye1", "f_contain", (W, H, ps), True)
    tiles, _ = fe.tile_plan()
    assert set((tiles["type"] & 3).tolist()) >= {0, 2} and np.isin(tiles["type"] & 3, (1, 3)).any()
    bg = bb.synthetic_background(W, H)
    table = rgba_table(11)
    for f in (fe, fe3):
        f.set_background(bg)
        f.set_rgba_table(table)
    bpp, pitch, y0 = (4 if rgba else 1), 1 << 26, 3
    d_faces = torch.randint(0, 256, (1, 6 * ps * ps), dtype=torch.uint8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    ref = Reference(torch, fe, bg, table if rgba else None)
    want = ref.frames(d_faces)[0]
    sentinel = torch.tensor(SENTINEL * 0x01010101 if rgba else SENTINEL, dtype=torch.int32 if rgba else torch.uint8, device="cuda")
    want_keep = torch.where(ref.valid.reshape(H, W), want, sentinel)
    screen = torch.empty((y0 + H, pitch), dtype=torch.uint8, device="cuda")
    for keep in (False, True):
        for ctx, x0, kernel_id in [(fe, 12, "ring"), (fe, 12, "K1"), (fe, 5, "K0"), (fe3, 12, "K3")]:
            screen.fill_(SENTINEL)
            ctx.set_kernel(1 if kernel_id == "K1" else 0)
            try:
                ctx.warp_view(d_faces, screen, x0=x0, y0=y0, nframes=1, keep_unmapped=keep, rgba=rgba)
            finally:
                ctx.set_kernel(0)
            torch.cuda.synchronize()
            k = ctx.last_kernel
            assert KERNEL[kernel_id] in k, (keep, kernel_id, k)
            rect = screen[y0:y0 + H, x0 * bpp:(x0 + W) * bpp]
            got = rect.contiguous().view(torch.int32) if rgba else rect
            assert torch.equal(got, want_keep if keep else want), (rgba, keep, kernel_id, k)
            # nothing outside the rectangle was written
            assert untouched(screen[:y0]) and untouched(screen[y0 + H:]), (rgba, keep, kernel_id, k)
            assert untouched(screen[y0:y0 + H, :x0 * bpp]) and untouched(screen[y0:y0 + H, (x0 + W) * bpp:]), (rgba, keep, kernel_id, k)
    screen.fill_(SENTINEL)
    with pytest.raises(bb.BlinkyError) as e:
        fe.warp_view(d_faces, screen, x0=0, y0=0, rowbytes=pitch + 16, nframes=1, rgba=rgba)
    assert e.value.code == bb.E_INVALID and "64 MB" in str(e.value)
    torch.cuda.synchronize()
    assert untouched(screen)


def untouched(region):
    """every byte of `region` (rows of a 4 GB screen) still holds the sentinel; one row at a time"""
    return not any(bool((row != SENTINEL).any()) for row in region)


# -- 6. frame count at the grid limit ---------------------------------------------------------------------------


def test_frame_count_at_the_grid_limit(bb, ctxs, torch_mod):
    """K0, K1 and K3 launch one grid row per frame (or group of frames), and gridDim.y is at most 65535: 65535 frames
    are warped, every one of them right, and 65536 are refused without a write."""
    torch = torch_mod
    fe, _ = ctxs
    W, H, ps = 64, 32, 16
    setup((fe,), "cube", "fisheye1", "f_contain", (W, H, ps), True)
    bg = bb.synthetic_background(W, H)
    fe.set_background(bg)
    n = 65535
    d_faces = torch.randint(0, 256, (n + 1, 6 * ps * ps), dtype=torch.uint8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    ref = Reference(torch, fe, bg)
    # this plan is all GATHER tiles: the default choice is K3 on its own
    runs = tiled_runs(fe, None)
    assert [r[2] for r in runs] == [KERNEL["K3"], KERNEL["K1"], KERNEL["K0"]]
    for ctx, how, kernel in runs:
        got, k = warp(torch, ctx, how, d_faces, n)
        assert kernel in k, (how, k)
        ref.check(d_faces, got, f"{n} frames, {how}: {k}")
        del got
    out = torch.full((n + 1, H, W), SENTINEL, dtype=torch.uint8, device="cuda")
    with pytest.raises(bb.BlinkyError) as e:
        fe.warp(d_faces, out, nframes=n + 1)
    assert e.value.code == bb.E_INVALID and "65535" in str(e.value)
    torch.cuda.synchronize()
    assert not bool((out != SENTINEL).any())


# -- 7. the forward builder over its cap of undecided grid points -----------------------------------------------

# lon/lat like equirect, through a loop whose bound is a libm result: the translated lens cannot show the bound
# exact, so the device leaves every grid point to the interpreter (the loop itself never runs)
UNDECIDED_LENS = """
map = "lens_forward"
max_fov = 360
max_vfov = 180
lens_width = 2*pi
lens_height = pi
onload = "f_contain"
function lens_forward(x, y, z)
  local lat, lon = ray_to_latlon(x, y, z)
  for k = 1, atan(1) do lat = lat + 1 end
  return lon, lat
end
"""


@pytest.mark.parametrize("ps", [400, 420])
def test_forward_builder_over_its_undecided_cap(bb, ctxs, palette, ps):
    """6 * 401^2 = 964806 grid points fit the device builder's 2^20 slots for undecided points and are all settled by
    the interpreter; 6 * 421^2 = 1063446 do not, and the device build gives up for the host's.  Either way the map,
    the display flags and the log are the single-threaded interpreter's."""
    fe, _ = ctxs
    W, H = 128, 64
    npoints = 6 * (ps + 1) ** 2
    with bb.Fisheye(device=None, palette=palette) as host:
        host.clear_log()
        setup((host,), "cube", "undecided", None, (W, H, ps), True, threads=1, lens_source=UNDECIDED_LENS)
        want_idx, want_tint = host.lensmap()
        want_display, want_log = host.display(), host.log
    fe.clear_log()
    setup((fe,), "cube", "undecided", None, (W, H, ps), True, threads=0, lens_source=UNDECIDED_LENS)
    info = fe.build_info
    if npoints <= 1 << 20:
        assert info.startswith(f"device (forward): {npoints} of {npoints} grid points re-evaluated"), info
    else:
        assert info.startswith(f"host (forward lens; too many grid points need the interpreter ({npoints}))"), info
    idx, tint = fe.lensmap()
    assert (idx >= 0).mean() > 0.9
    assert np.array_equal(idx, want_idx) and np.array_equal(tint, want_tint)
    assert fe.display() == want_display and fe.log == want_log
