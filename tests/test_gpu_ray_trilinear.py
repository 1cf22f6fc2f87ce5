"""The trilinear warp from a ray field (blinky_warp_device_rays_trilinear, warp_rays(filter="trilinear")) on the GPU, every
byte of each output buffer and of the scratch's pyramids against tests/ray_trilinear_reference.py (the host set_raymap for
mapping and plate, the ray_texel.h shim for footprint, level, weight and positions, numpy for the pyramid, taps, blends
and the mix of levels), margins included."""
import numpy as np
import pytest

import ray_bilinear_reference as br
import ray_trilinear_reference as tr
from test_gpu_ray_supersample import TABLE, faces_for, field, install, setup
from test_gpu_ray_warp import Screens, layouts, matrices, yaw

pytestmark = pytest.mark.gpu

W, H = 96, 64
PS = 97           # panini f_fov 180 on a 96 x 64 view: levels 0, 1 and 2 all occur, and every level's size is odd
SENTINEL = 0xA5   # the scratch's bytes before a call


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return tr.compile_shim(tmp_path_factory.mktemp("trilinear_gpu"))


@pytest.fixture()
def fe(bb, palette, cuda_device):
    c = bb.Fisheye(device=cuda_device, palette=palette)
    yield c
    c.close()


@pytest.fixture()
def globe(bb, palette, shim):
    made = []

    def make(name="cube", rubix=False, grid=None):
        made.append(tr.TrilinearGlobe(bb, palette, name, shim, rubix, grid))
        return made[-1]

    yield make
    for g in made:
        g.close()


def prepare(fe, ps=PS, **kw):
    """setup() at plate size ps: the background"""
    bg = setup(fe, **kw)
    layout = kw.get("layout")
    install(fe, W, H, bg, ps)
    if layout:
        fe.set_face_layout(*layout)
    return bg


def scratch_for(torch, fe, n, extra=4096):
    B = fe.ray_pyramid_bytes()
    return torch.full((n * B + extra,), SENTINEL, dtype=torch.uint8, device="cuda"), B


def run(torch, fe, d_faces, d_rays, d_x, scr, n, keep, tables=None, scratch=None):
    out = scr.new()
    launches = fe.launch_count
    fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=scr.x0, y0=scr.y0, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep, rgba=True,
                 tables=tables, screen_stride=scr.stride, filter="trilinear", scratch=scratch)
    torch.cuda.synchronize()
    lmax = len(tr.level_sizes(fe.platesize)) - 1
    assert fe.launch_count == launches + lmax + 1
    return out, fe.last_kernel


def expected(torch, g, scr, bg, d_faces, d_rays, d_x, n, keep, tables=None, layout=None, ps=PS, w=W, h=H):
    """(the screens scr.fill with the view rectangles of n frames written by the rule, [each frame's pyramid bytes])"""
    faces = d_faces.cpu().numpy() if d_faces.numel() < (1 << 28) else d_faces
    fields = d_rays.cpu().numpy()
    xs = None if d_x is None else d_x.cpu().numpy()
    tabs = None if tables is None else tables.cpu().numpy().view(np.uint32)
    exp = scr.fill.clone()
    pyramids = []
    for f in range(n):
        fld = fields if fields.ndim == 3 else fields[f]
        M = None if xs is None else (xs if xs.ndim == 2 else xs[f])
        tab = TABLE if tabs is None else (tabs if tabs.ndim == 1 else tabs[f])
        fc = faces.reshape(faces.shape[0], -1)[min(f, faces.shape[0] - 1)] if isinstance(faces, np.ndarray) else faces[min(f, faces.shape[0] - 1)]
        pix, written, levels, _, _ = g.frame(fld, M, fc, bg.reshape(h, w), ps, layout=layout, table=tab)
        pyramids.append(g.scratch_bytes(levels))
        v = exp.as_strided((h, w, 4), (scr.rowbytes, 4, 1), f * scr.stride + scr.y0 * scr.rowbytes + 4 * scr.x0)
        new = torch.from_numpy(pix).cuda()
        v.copy_(new.where(torch.from_numpy(written).cuda()[..., None], v) if keep else new)
    return exp, pyramids


def assert_scratch(scratch, B, pyramids):
    """each frame's pyramid where the layout puts it; the rounding, and every byte past the frames, untouched"""
    got = scratch.cpu().numpy()
    for f, want in enumerate(pyramids):
        frame = got[f * B:(f + 1) * B]
        bad = np.nonzero(frame[: len(want)] != want)[0]
        assert bad.size == 0, (f, bad.size, bad[:8].tolist())
        assert (frame[len(want):] == SENTINEL).all(), f
    assert (got[len(pyramids) * B:] == SENTINEL).all()


def check(torch, fe, g, bg, d_faces, d_rays, d_x, scr, n, keep, tables=None, layout=None, expect_kernel=None, ps=PS):
    scratch, B = scratch_for(torch, fe, n)
    got, kernel = run(torch, fe, d_faces, d_rays, d_x, scr, n, keep, tables, scratch)
    if expect_kernel:
        assert kernel.startswith(expect_kernel), kernel
    want, pyramids = expected(torch, g, scr, bg, d_faces, d_rays, d_x, n, keep, tables, layout, ps)
    bad = (got != want).nonzero().flatten()
    assert bad.numel() == 0, (kernel, bad.numel(), bad[:8].tolist())
    assert_scratch(scratch, B, pyramids)
    return got, kernel


def levels_seen(fe, g, d_rays, M, ps=PS, w=W, h=H):
    p = br.params(g.fe, w, h, ps, g.grid)
    s, rho2 = tr.header_trilinear(g.lib, p, M, d_rays.cpu().numpy(), len(tr.level_sizes(ps)) - 1)
    m = s[:, 0] == 1
    return set(s[m, 2].tolist()), s, rho2


# ---- every kernel instance against the rule ----------------------------------------------------------------------

@pytest.mark.parametrize("tables", ["context", "frames"])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("rubix", [False, True])
def test_every_instance_follows_the_rule(torch, fe, globe, rubix, keep, tables):
    bg = prepare(fe, rubix=rubix)
    g = globe(rubix=rubix)
    n = 3
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    d_x = torch.from_numpy(np.stack([yaw(0), yaw(29), yaw(-71)])).cuda()
    d_tables = None
    if tables == "frames":
        d_tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=3, y0=5, extra=13)
    tag = f"ray_trilinear_kernel<rubix={int(rubix)},keep={int(keep)},tables={int(tables == 'frames')}>"
    seen, s, _ = levels_seen(fe, g, d_rays, yaw(29))
    assert {0, 1, 2} <= seen and (s[s[:, 0] == 1, 3] > 0).any(), sorted(seen)
    check(torch, fe, g, bg, faces_for(torch, fe, n, ps=PS), d_rays, d_x, scr, n, keep, d_tables, expect_kernel=tag)


# ---- properties of the rule --------------------------------------------------------------------------------------

def test_footprint_below_one_texel_equals_bilinear(torch, fe, globe):
    """rectilinear f_fov 30 on 48^2 plates magnifies everywhere (rho < 1 at every mapped pixel, checked through the
    shim): the output equals blinky_warp_device_rays_bilinear at k = 1 byte for byte"""
    ps = 48
    fe.command("f_globe cube")
    fe.command("f_lens rectilinear")
    fe.command("f_fov 30")
    fe.set_rgba_table(TABLE)
    bg = np.random.default_rng(1).integers(0, 256, W * H, dtype=np.uint8)
    install(fe, W, H, bg, ps)
    d_rays = torch.from_numpy(fe.raymap(W, H)).cuda()
    n = 3
    d_x = torch.from_numpy(np.stack([yaw(10), yaw(100), yaw(-45)])).cuda()
    g = globe()
    for f in range(n):
        seen, s, rho2 = levels_seen(fe, g, d_rays, d_x[f].cpu().numpy(), ps)
        assert seen == {0} and (rho2[s[:, 0] == 1] < 1).all() and (s[:, 0] == 1).mean() > 0.9
    d_faces = faces_for(torch, fe, n, ps=ps)
    outs = []
    for filt in ("trilinear", "bilinear"):
        out = torch.zeros((n, H, W, 4), dtype=torch.uint8, device="cuda")
        fe.warp_rays(d_faces, out, d_rays, d_x, rowbytes=4 * W, screen_stride=4 * W * H, rgba=True, filter=filt)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), int((outs[0] != outs[1]).sum())


def test_one_colour_plates_stay_that_colour(torch, fe):
    """faces whose plates are each one byte (rubix off): every level of a plate is its colour, so the output is the
    nearest warp's"""
    prepare(fe)
    n = 2
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    plates = np.array([[11, 60, 99, 140, 201, 250], [3, 77, 128, 180, 9, 33]], np.uint8)[:, : fe.numplates]
    d_faces = torch.from_numpy(np.repeat(plates, PS * PS, axis=1)).cuda()
    for keep in (False, True):
        scr = Screens(torch, n, True, x0=2, y0=3, extra=9)
        got, _ = run(torch, fe, d_faces, d_rays, d_x, scr, n, keep)
        near = scr.new()
        fe.warp_rays(d_faces, near.data_ptr(), d_rays, d_x, x0=2, y0=3, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep, rgba=True,
                     screen_stride=scr.stride)
        torch.cuda.synchronize()
        assert torch.equal(got, near), (keep, int((got != near).sum()))


def test_keep_writes_the_pixels_of_the_nearest_warp(torch, fe):
    prepare(fe, rubix=True)
    n = 3
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    d_faces = faces_for(torch, fe, n, ps=PS)

    def written(filt):
        outs = []
        for fill in (0, 255):
            out = torch.full((n, H, W, 4), fill, dtype=torch.uint8, device="cuda")
            fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, rowbytes=4 * W, screen_stride=4 * W * H, nframes=n, keep_unmapped=True, rgba=True,
                         filter=filt)
            outs.append(out)
        torch.cuda.synchronize()
        return (outs[0] == outs[1]).all(-1)

    near, tri = written("nearest"), written("trilinear")
    assert bool(near.any()) and not bool(near.all())
    assert torch.equal(near, tri), int((near != tri).sum())


# ---- plate sizes, face layouts -----------------------------------------------------------------------------------

@pytest.mark.parametrize("ps", [1, 97, 6688])
def test_plate_sizes(torch, fe, globe, ps):
    """1 (no pyramid: B = 0, a NULL scratch is taken), 97 (odd sizes on every level), 6688 (13 levels)"""
    bg = prepare(fe, ps=ps, rubix=ps == 97)
    g = globe(rubix=ps == 97)
    n = 1 if ps == 6688 else 2
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    d_faces = faces_for(torch, fe, n, ps=ps) if ps < 6688 else torch.randint(0, 256, (1, 6 * ps * ps), dtype=torch.uint8, device="cuda")
    B = fe.ray_pyramid_bytes()
    assert B == tr.pyramid_layout(ps, fe.numplates)[2]
    if ps == 1:
        assert B == 0
        lib = fe._lib
        out = torch.zeros((n, H, W, 4), dtype=torch.uint8, device="cuda")
        assert lib.blinky_warp_device_rays_trilinear(fe._ctx, d_faces.data_ptr(), d_faces.stride(0), d_rays.data_ptr(), 0, d_x.data_ptr(), 36,
                                                     out.data_ptr(), 4 * W * H, 4 * W, 0, 0, n, 0, None, 0, None, 0, None) == 0
        torch.cuda.synchronize()
        assert fe.last_kernel.endswith("levels=0")
    seen, _, _ = levels_seen(fe, g, d_rays, d_x[0].cpu().numpy(), ps)
    if ps == 6688:
        assert max(seen) >= 6, sorted(seen)
    check(torch, fe, g, bg, d_faces, d_rays, d_x, Screens(torch, n, True, x0=1, y0=2, extra=3), n, False, ps=ps)


SENTINEL_BYTE = 255


def test_tight_atlas_never_shows_its_margin(torch, fe, globe):
    """plates packed edge to edge with a sentinel byte in the rows and columns around them (rubix off): neither the
    pyramid nor the level-0 taps cross into a neighbouring plate or the margin, so the sentinel colour (alpha 0; every
    other colour has alpha 255) never appears, and every byte follows the rule"""
    ps = PS
    rowbytes = 3 * ps + 2
    lay = (rowbytes, [(1, 1), (1 + ps, 1), (1 + 2 * ps, 1), (1, 1 + ps), (1 + ps, 1 + ps), (1 + 2 * ps, 1 + ps)])
    table = np.array([b | (255 - b) << 8 | (b * 7 % 256) << 16 | 0xFF000000 for b in range(256)], np.uint32)
    table[SENTINEL_BYTE] = 0x00FF00FF
    bg = prepare(fe, layout=lay) % SENTINEL_BYTE
    fe.set_background(bg)
    g = globe()
    n = 2
    rng = np.random.default_rng(5)
    atlas = np.full((n, 2 * ps + 2, rowbytes), SENTINEL_BYTE, np.uint8)
    atlas[:, 1:-1, 1:-1] = rng.integers(0, SENTINEL_BYTE, (n, 2 * ps, 3 * ps), dtype=np.uint8)
    d_faces = torch.from_numpy(atlas).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    d_tab = torch.from_numpy(table.view(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=1, y0=2, extra=3)
    got, _ = check(torch, fe, g, bg, d_faces, torch.from_numpy(field(fe, 1)).cuda(), d_x, scr, n, False, d_tab, layout=lay)
    view = got.as_strided((n, H, W, 4), (scr.stride, scr.rowbytes, 4, 1), scr.y0 * scr.rowbytes + 4 * scr.x0)
    assert bool((view[..., 3] == 255).all())


@pytest.mark.parametrize("name", ["atlas", "odd"])
def test_face_layouts(torch, fe, globe, name):
    rowbytes, origins = layouts()[name]
    # layouts() is at plate size 48: scale the origins to this test's plates
    lay = (rowbytes // 48 * PS + rowbytes % 48, [(x // 48 * PS + x % 48, y // 48 * PS + y % 48) for x, y in origins])
    bg = prepare(fe, rubix=True, grid=(4, 3.0, 2.0), layout=lay)
    g = globe(rubix=True, grid=(4, 3.0, 2.0))
    n = 2
    check(torch, fe, g, bg, faces_for(torch, fe, n, lay, ps=PS), torch.from_numpy(field(fe, 1)).cuda(), torch.from_numpy(matrices(n)).cuda(),
          Screens(torch, n, True, x0=5, y0=1, extra=7), n, True, layout=lay)


# ---- transform forms and batches ---------------------------------------------------------------------------------

def test_per_frame_fields_matrices_and_tables(torch, fe, globe):
    bg = prepare(fe, rubix=True)
    g = globe(rubix=True)
    n = 3
    base = field(fe, 1)
    fields = np.stack([base, base[:, ::-1].copy(), np.random.default_rng(12).normal(size=base.shape).astype(np.float32)])
    d_faces = faces_for(torch, fe, n, ps=PS)
    tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=1, y0=2, extra=11)
    _, kernel = check(torch, fe, g, bg, d_faces, torch.from_numpy(fields).cuda(), torch.from_numpy(matrices(n)).cuda(), scr, n, False, tables)
    assert "frames/thread=1" in kernel, kernel
    check(torch, fe, g, bg, d_faces, torch.from_numpy(fields).cuda(), None, scr, n, True)
    # one field, one matrix, several frames: the sample is carried from frame to frame
    _, kernel = check(torch, fe, g, bg, d_faces, torch.from_numpy(base).cuda(), torch.from_numpy(matrices(5)[4]).cuda(), scr, n, True, tables)


@pytest.mark.parametrize("globe_name", ["tetra", "trism", "cube_edge", "cube_corner"])
def test_other_argmax_globes(torch, fe, globe, globe_name):
    bg = prepare(fe, globe=globe_name, rubix=True)
    g = globe(globe_name, rubix=True)
    n = 2
    check(torch, fe, g, bg, faces_for(torch, fe, n, ps=PS), torch.from_numpy(field(fe, 1)).cuda(),
          torch.from_numpy(matrices(n, seed=len(globe_name))).cuda(), Screens(torch, n, True, x0=0, y0=0, extra=0), n, False)


def test_4k_look_around(torch, fe, globe):
    """fisheye1 f_contain at 3840 x 2160 on 2048^2 plates, two frames of one exported field with per-frame yaws"""
    w, h, ps = 3840, 2160, 2048
    fe.command("f_globe cube")
    fe.command("f_lens fisheye1")
    fe.command("f_contain")
    fe.set_rgba_table(TABLE)
    bg = np.random.default_rng(3).integers(0, 256, w * h, dtype=np.uint8)
    install(fe, w, h, bg, ps)
    d_rays = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    fe.raymap(w, h, out=d_rays)
    n = 2
    d_x = torch.from_numpy(np.stack([yaw(5), yaw(-40)])).cuda()
    d_faces = faces_for(torch, fe, n, ps=ps)
    scratch, B = scratch_for(torch, fe, n)
    out = torch.full((n, h, w, 4), 3, dtype=torch.uint8, device="cuda")
    fe.warp_rays(d_faces, out, d_rays, d_x, rowbytes=4 * w, screen_stride=4 * w * h, rgba=True, filter="trilinear", scratch=scratch)
    torch.cuda.synchronize()
    g = globe()
    fields = d_rays.cpu().numpy()
    pyr = []
    for f in range(n):
        pix, _, levels, s, _ = g.frame(fields, d_x[f].cpu().numpy(), d_faces[f].cpu().numpy(), bg.reshape(h, w), ps, table=TABLE)
        assert len(set(s[s[:, 0] == 1, 2].tolist())) >= 3
        assert np.array_equal(out[f].cpu().numpy(), pix), f
        pyr.append(g.scratch_bytes(levels))
    assert_scratch(scratch, B, pyr)


# ---- context state, graphs and refusals --------------------------------------------------------------------------

def test_the_context_does_not_change(torch, fe):
    prepare(fe, rubix=True)
    fe.command("f_lens stereographic")
    fe.build_lensmap(W, H, PS, threads=1)
    state = lambda: (fe.lensmap_packed().tobytes(), fe.display(), fe.build_info, fe.needs_rebuild(W, H, PS), fe.plan_digest(),  # noqa: E731
                     fe.mapped_pixels, fe.width, fe.height, fe.platesize, fe.ray_pyramid_bytes())
    fe.command("f_lens panini")
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    fe.command("f_lens stereographic")
    before = state()
    out = torch.zeros(2 * W * H * 4, dtype=torch.uint8, device="cuda")
    fe.warp_rays(faces_for(torch, fe, 2, ps=PS), out.data_ptr(), d_rays, torch.from_numpy(matrices(2)).cuda(), rowbytes=4 * W,
                 screen_stride=4 * W * H, rgba=True, filter="trilinear")
    torch.cuda.synchronize()
    assert fe.last_kernel.startswith("ray_trilinear_kernel<")
    assert state() == before


def test_graph_replay_reads_new_matrices_tables_and_faces(torch, fe, globe):
    bg = prepare(fe, rubix=True)
    g = globe(rubix=True)
    n = 3
    d_faces = faces_for(torch, fe, n, ps=PS)
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=6, y0=3, extra=5)
    scratch, B = scratch_for(torch, fe, n)
    out = scr.new()
    # a capture cannot allocate the scratch
    with pytest.raises(ValueError, match="persistent scratch"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=6, y0=3, rowbytes=scr.rowbytes, nframes=n, rgba=True, tables=tables,
                         screen_stride=scr.stride, filter="trilinear")
    launches = fe.launch_count
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=6, y0=3, rowbytes=scr.rowbytes, nframes=n, rgba=True, tables=tables,
                     screen_stride=scr.stride, filter="trilinear", scratch=scratch)
    assert fe.launch_count == launches + len(tr.level_sizes(PS))
    d_x.copy_(torch.from_numpy(np.stack([yaw(123.0), yaw(-40.0), yaw(7.0)])))
    tables[1].copy_(torch.from_numpy(np.random.default_rng(9).integers(0, 2**31, 256).astype(np.int32)))
    d_faces.copy_(faces_for(torch, fe, n, seed=11, ps=PS))
    out.copy_(scr.fill)
    graph.replay()
    torch.cuda.synchronize()
    replayed, replayed_scratch = out.clone(), scratch.clone()
    want, pyramids = expected(torch, g, scr, bg, d_faces, d_rays, d_x, n, False, tables)
    assert torch.equal(replayed, want), int((replayed != want).sum())
    assert_scratch(replayed_scratch, B, pyramids)
    # the eager call gives the same bytes
    eager, _ = run(torch, fe, d_faces, d_rays, d_x, scr, n, False, tables, scratch)
    assert torch.equal(eager, replayed)
    del graph
    fe.release_captures()


def test_refusals_launch_nothing(bb, torch, fe, palette, cuda_device):
    lib = bb.load_library()
    prepare(fe)
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    d_x = torch.from_numpy(matrices(2)).cuda()
    d_faces = faces_for(torch, fe, 2, ps=PS)
    tab = torch.zeros(2 * 256 + 4, dtype=torch.int32, device="cuda")
    out = torch.zeros(2 * W * H * 4 + 16, dtype=torch.uint8, device="cuda")
    B = fe.ray_pyramid_bytes()
    scratch = torch.full((2 * B + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    R, X, F, O, T, S = d_rays.data_ptr(), d_x.data_ptr(), d_faces.data_ptr(), out.data_ptr(), tab.data_ptr(), scratch.data_ptr()

    def call(rays=R, rstride=0, xstride=36, o=O, rowbytes=4 * W, tables=None, tstride=0, s=S, sbytes=2 * B, ctx=None):
        return lib.blinky_warp_device_rays_trilinear(fe._ctx if ctx is None else ctx, F, d_faces.stride(0), rays, rstride, X, xstride, o,
                                                     4 * W * H, rowbytes, 0, 0, 2, 0, tables, tstride, s, sbytes, None)

    assert call() == bb.OK and call(tables=T, tstride=1024) == bb.OK
    torch.cuda.synchronize()
    launches, kernel = fe.launch_count, fe.last_kernel
    scratch.fill_(SENTINEL)
    out.zero_()
    cases = [("ray_stride short by one ray", dict(rstride=12 * W * H - 12)), ("ray_stride not a multiple of 4", dict(rstride=12 * W * H + 2)),
             ("xform_stride short", dict(xstride=32)), ("rays misaligned", dict(rays=R + 2)), ("screen misaligned", dict(o=O + 2)),
             ("rowbytes misaligned", dict(rowbytes=4 * W + 2)), ("rowbytes short", dict(rowbytes=4 * W - 4)),
             ("tables misaligned", dict(tables=T + 4)), ("table_stride", dict(tables=T, tstride=1008)), ("NULL rays", dict(rays=None)),
             ("NULL screen", dict(o=None)), ("NULL scratch", dict(s=None)), ("scratch misaligned", dict(s=S + 8)),
             ("scratch short by a byte", dict(sbytes=2 * B - 1))]
    for what, kw in cases:
        assert call(**kw) == bb.E_INVALID, what
    assert fe.launch_count == launches and fe.last_kernel == kernel
    fe.command("f_globe fast")
    assert call() == bb.E_STATE and "blinky_set_raymap_device" in lib.blinky_last_error(fe._ctx).decode()
    assert fe.launch_count == launches
    torch.cuda.synchronize()
    assert bool((scratch == SENTINEL).all()) and bool((out == 0).all())
    fresh = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        fresh.command("f_globe cube")
        assert call(ctx=fresh._ctx) == bb.E_STATE, "no lensmap installed"
        with pytest.raises(bb.BlinkyError) as e:
            fresh.ray_pyramid_bytes()
        assert e.value.code == bb.E_STATE
        assert fresh.launch_count == 0
    finally:
        fresh.close()


# ---- quality -----------------------------------------------------------------------------------------------------

def test_iid_noise_shimmers_less_than_nearest(torch, fe):
    """fisheye1 f_contain minifies 512^2 plates of iid noise on a 320 x 180 view: under a 0.1 degree yaw step the mean
    absolute frame-to-frame change of trilinear is under half of nearest's, and trilinear is closer than nearest to the
    k = 4 supersampled image"""
    w, h, ps, k = 320, 180, 512, 4
    fe.command("f_globe cube")
    fe.command("f_lens fisheye1")
    fe.command("f_contain")
    grey = np.array([b | b << 8 | b << 16 | 0xFF000000 for b in range(256)], np.uint32)
    fe.set_rgba_table(grey)
    fe.build_lensmap(w, h, ps, threads=0)   # the view's size; its mapped pixels are the disc at any yaw
    base = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    fe.raymap(w, h, out=base)
    big = torch.empty((k * h, k * w, 3), dtype=torch.float32, device="cuda")
    fe.raymap(k * w, k * h, out=big)
    d_x = torch.from_numpy(np.stack([yaw(30.0), yaw(30.1)])).cuda()
    d_faces = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (1, 6 * ps * ps), dtype=np.uint8)).cuda()

    def render(filt, rays, ss=1):
        out = torch.zeros((2, h, w, 4), dtype=torch.uint8, device="cuda")
        fe.warp_rays(d_faces, out, rays, d_x, rowbytes=4 * w, screen_stride=4 * w * h, rgba=True, face_stride=0, filter=filt, supersample=ss)
        return out[..., 0].to(torch.float32)

    near, tri, ref = render("nearest", base), render("trilinear", base), render("nearest", big, k)
    torch.cuda.synchronize()
    mask = torch.from_numpy(fe.lensmap()[0].reshape(h, w) >= 0).cuda()
    assert int(mask.sum()) > w * h // 3   # the disc

    def shimmer(a):
        return float((a[1] - a[0]).abs()[mask].mean())

    def err(a):
        return float((a[0] - ref[0]).abs()[mask].mean())

    assert shimmer(tri) < 0.5 * shimmer(near), (shimmer(tri), shimmer(near))
    assert err(tri) < err(near), (err(tri), err(near))
