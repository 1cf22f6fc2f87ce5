"""The bilinear warp from a ray field (blinky_warp_device_rays_bilinear, warp_rays(filter="bilinear")) on the GPU, every
byte of each output buffer against tests/ray_bilinear_reference.py (the host set_raymap for mapping and plate, the
ray_texel.h shim for positions, numpy for taps, LUTs, tables, blend and average), margins included."""
import numpy as np
import pytest

import ray_bilinear_reference as br
import ray_reference as rr
from test_gpu_ray_supersample import TABLE, faces_for, field, install, setup
from test_gpu_ray_warp import Screens, layouts, matrices, yaw

pytestmark = pytest.mark.gpu

W, H, PS = 96, 64, 48


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return br.compile_shim(tmp_path_factory.mktemp("bilinear_gpu"))


@pytest.fixture()
def fe(bb, palette, cuda_device):
    c = bb.Fisheye(device=cuda_device, palette=palette)
    yield c
    c.close()


@pytest.fixture()
def globe(bb, palette, shim):
    made = []

    def make(name="cube", rubix=False, grid=None):
        made.append(br.BilinearGlobe(bb, palette, name, shim, rubix, grid))
        return made[-1]

    yield make
    for g in made:
        g.close()


def run(torch, fe, k, d_faces, d_rays, d_x, scr, n, keep, tables=None, **kw):
    out = scr.new()
    launches = fe.launch_count
    fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=scr.x0, y0=scr.y0, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep, rgba=True,
                 tables=tables, screen_stride=scr.stride, supersample=k, filter="bilinear", **kw)
    torch.cuda.synchronize()
    assert fe.launch_count == launches + 1
    return out, fe.last_kernel


def expected(torch, g, scr, k, bg, d_faces, d_rays, d_x, n, keep, tables=None, layout=None, w=W, h=H, ps=PS):
    """the screens scr.fill with the view rectangles of n frames written by the rule"""
    faces = d_faces.cpu().numpy() if d_faces.numel() < (1 << 28) else d_faces
    fields = d_rays.cpu().numpy()
    xs = None if d_x is None else d_x.cpu().numpy()
    tabs = None if tables is None else tables.cpu().numpy().view(np.uint32)
    exp = scr.fill.clone()
    for f in range(n):
        fld = fields if fields.ndim == 3 else fields[f]
        M = None if xs is None else (xs if xs.ndim == 2 else xs[f])
        tab = TABLE if tabs is None else (tabs if tabs.ndim == 1 else tabs[f])
        fc = faces.reshape(faces.shape[0], -1)[min(f, faces.shape[0] - 1)]
        pix, written = g.frame(fld, M, fc, bg.reshape(h, w), k, ps, layout=layout, table=tab)
        v = exp.as_strided((h, w, 4), (scr.rowbytes, 4, 1), f * scr.stride + scr.y0 * scr.rowbytes + 4 * scr.x0)
        new = torch.from_numpy(pix).cuda()
        v.copy_(new.where(torch.from_numpy(written).cuda()[..., None], v) if keep else new)
    return exp


def check(torch, fe, g, k, bg, d_faces, d_rays, d_x, scr, n, keep, tables=None, layout=None, expect_kernel=None):
    got, kernel = run(torch, fe, k, d_faces, d_rays, d_x, scr, n, keep, tables)
    if expect_kernel:
        assert kernel.startswith(expect_kernel), kernel
    want = expected(torch, g, scr, k, bg, d_faces, d_rays, d_x, n, keep, tables, layout)
    bad = (got != want).nonzero().flatten()
    assert bad.numel() == 0, (kernel, bad.numel(), bad[:8].tolist())
    return got, kernel


# ---- every kernel instance against the rule ----------------------------------------------------------------------

@pytest.mark.parametrize("tables", ["context", "frames"])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("rubix", [False, True])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_every_instance_follows_the_rule(torch, fe, globe, k, rubix, keep, tables):
    bg = setup(fe, rubix=rubix)
    g = globe(rubix=rubix)
    n = 3
    d_rays = torch.from_numpy(field(fe, k)).cuda()
    d_x = torch.from_numpy(np.stack([yaw(0), yaw(29), yaw(-71)])).cuda()
    d_tables = None
    if tables == "frames":
        d_tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=3, y0=5, extra=13)
    tag = f"ray_bilinear_kernel<k={k},rubix={int(rubix)},keep={int(keep)},tables={int(tables == 'frames')}>"
    check(torch, fe, g, k, bg, faces_for(torch, fe, n), d_rays, d_x, scr, n, keep, d_tables, expect_kernel=tag)


# ---- against the nearest warps -----------------------------------------------------------------------------------

def test_k1_keep_writes_the_pixels_of_the_nearest_warp(torch, fe):
    setup(fe, rubix=True)
    n = 3
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    d_faces = faces_for(torch, fe, n)

    def written(bilinear):
        outs = []
        for fill in (0, 255):
            out = torch.full((n, H, W, 4), fill, dtype=torch.uint8, device="cuda")
            fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, rowbytes=4 * W, screen_stride=4 * W * H, nframes=n, keep_unmapped=True, rgba=True,
                         filter="bilinear" if bilinear else "nearest")
            outs.append(out)
        torch.cuda.synchronize()
        return (outs[0] == outs[1]).all(-1)

    near, bil = written(False), written(True)
    assert bool(near.any()) and not bool(near.all())
    assert torch.equal(near, bil), int((near != bil).sum())


@pytest.mark.parametrize("k", [1, 2, 3])
def test_one_byte_per_plate_equals_nearest(torch, fe, k):
    """faces whose plates are each one byte (rubix off): every tap of a sample has its texel's colour, so the bilinear
    warp gives the nearest warp's output exactly"""
    setup(fe, rubix=False)
    n = 2
    d_rays = torch.from_numpy(field(fe, k)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    plates = np.array([[11, 60, 99, 140, 201, 250], [3, 77, 128, 180, 9, 33]], np.uint8)[:, : fe.numplates]
    d_faces = torch.from_numpy(np.repeat(plates, PS * PS, axis=1)).cuda()
    for keep in (False, True):
        scr = Screens(torch, n, True, x0=2, y0=3, extra=9)
        got, _ = run(torch, fe, k, d_faces, d_rays, d_x, scr, n, keep)
        near = scr.new()
        fe.warp_rays(d_faces, near.data_ptr(), d_rays, d_x, x0=2, y0=3, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep, rgba=True,
                     screen_stride=scr.stride, supersample=k)
        torch.cuda.synchronize()
        assert torch.equal(got, near), (k, keep, int((got != near).sum()))


def test_magnified_view_is_smoother_than_nearest(torch, fe, globe):
    """rectilinear f_fov 30 on 48^2 plates: each texel covers several pixels, so bilinear output differs from nearest
    and its largest step between neighbouring pixels is smaller"""
    fe.command("f_globe cube")
    fe.command("f_lens rectilinear")
    fe.command("f_fov 30")
    grey = np.array([b | b << 8 | b << 16 | 0xFF000000 for b in range(256)], np.uint32)
    fe.set_rgba_table(grey)
    bg = np.zeros(W * H, np.uint8)
    install(fe, W, H, bg)
    d_rays = torch.from_numpy(fe.raymap(W, H)).cuda()
    d_x = torch.from_numpy(yaw(10)).cuda()
    d_faces = faces_for(torch, fe, 1)
    outs = []
    for filt in ("nearest", "bilinear"):
        out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, rowbytes=4 * W, rgba=True, filter=filt)
        outs.append(out)
    torch.cuda.synchronize()
    near, bil = (o[..., 0].to(torch.int32) for o in outs)
    assert not torch.equal(near, bil)

    def step(a):
        return max(int((a[:, 1:] - a[:, :-1]).abs().max()), int((a[1:] - a[:-1]).abs().max()))

    assert step(bil) < step(near), (step(bil), step(near))
    pix, _ = globe().frame(d_rays.cpu().numpy(), yaw(10), d_faces[0].cpu().numpy(), bg.reshape(H, W), 1, PS, table=grey)
    assert np.array_equal(outs[1].cpu().numpy(), pix)


@pytest.mark.parametrize("k", [2, 3, 4])
def test_k_is_the_box_average_of_k1(torch, fe, k):
    """frame f at k = the k x k box average of the k = 1 bilinear warp at k W x k H, background repeated k x k"""
    bg = setup(fe, rubix=True)
    n = 3
    d_rays = torch.from_numpy(field(fe, k)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    d_faces = faces_for(torch, fe, n)
    tables = torch.from_numpy(np.random.default_rng(6).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    out = torch.zeros((n, H, W, 4), dtype=torch.uint8, device="cuda")
    fe.warp_rays(d_faces, out, d_rays, d_x, rowbytes=4 * W, screen_stride=4 * W * H, rgba=True, tables=tables, supersample=k, filter="bilinear")
    install(fe, k * W, k * H, np.repeat(np.repeat(bg.reshape(H, W), k, 0), k, 1))
    big = torch.zeros((n, k * H, k * W, 4), dtype=torch.uint8, device="cuda")
    fe.warp_rays(d_faces, big, d_rays, d_x, rowbytes=4 * k * W, screen_stride=4 * k * k * W * H, rgba=True, tables=tables, filter="bilinear")
    assert fe.last_kernel.startswith("ray_bilinear_kernel<k=1,"), fe.last_kernel
    s = big.view(n, H, k, W, k, 4).to(torch.int32).sum((2, 4))
    avg = ((s + k * k // 2) // (k * k)).to(torch.uint8)
    torch.cuda.synchronize()
    assert torch.equal(out, avg), int((out != avg).sum())


# ---- face layouts, plate size limit ------------------------------------------------------------------------------

SENTINEL_BYTE = 255


@pytest.mark.parametrize("k", [1, 2])
def test_tight_atlas_never_reads_outside_a_plate(torch, fe, globe, k):
    """plates packed edge to edge in an atlas with a sentinel byte in the rows and columns around them (rubix off, so
    that no LUT can produce the byte): no tap crosses into a neighbouring plate or the margin, so the sentinel colour
    (alpha 0; every other colour has alpha 255) never appears, and every byte follows the rule"""
    ps = PS
    rowbytes = 3 * ps + 2
    lay = (rowbytes, [(1, 1), (1 + ps, 1), (1 + 2 * ps, 1), (1, 1 + ps), (1 + ps, 1 + ps), (1 + 2 * ps, 1 + ps)])
    table = np.array([b | (255 - b) << 8 | (b * 7 % 256) << 16 | 0xFF000000 for b in range(256)], np.uint32)
    table[SENTINEL_BYTE] = 0x00FF00FF
    bg = setup(fe, layout=lay) % SENTINEL_BYTE
    fe.set_background(bg)
    g = globe()
    n = 2
    rng = np.random.default_rng(5)
    atlas = np.full((n, 2 * ps + 2, rowbytes), SENTINEL_BYTE, np.uint8)
    atlas[:, 1:-1, 1:-1] = rng.integers(0, SENTINEL_BYTE, (n, 2 * ps, 3 * ps), dtype=np.uint8)
    d_faces = torch.from_numpy(atlas).cuda()
    d_rays = torch.from_numpy(field(fe, k)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    d_tab = torch.from_numpy(table.view(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=1, y0=2, extra=3)
    got, kernel = run(torch, fe, k, d_faces, d_rays, d_x, scr, n, False, d_tab)
    want = expected(torch, g, scr, k, bg, d_faces, d_rays, d_x, n, False, d_tab, layout=lay)
    assert torch.equal(got, want), (kernel, int((got != want).sum()))
    view = got.as_strided((n, H, W, 4), (scr.stride, scr.rowbytes, 4, 1), scr.y0 * scr.rowbytes + 4 * scr.x0)
    assert bool((view[..., 3] == 255).all())


def test_plate_size_6688_clamps_taps_at_6687(torch, fe, globe):
    """rays at texel centres and plate edges of 6688^2 plates: taps at -1 and 6688 are clamped to 0 and 6687"""
    ps = 6688
    fe.command("f_globe cube")
    fe.set_rubix(True)
    fe.set_rgba_table(TABLE)
    w, h = 64, 32
    bg = np.random.default_rng(2).integers(0, 256, w * h, dtype=np.uint8)
    fe.set_lensmap(np.full((h, w), 0x70000000, np.uint32), ps, fe.numplates)
    fe.set_background(bg)
    plates = fe.plates()
    rng = np.random.default_rng(8)
    edge = np.array([0.0, 0.2 / ps, 0.5 / ps, 1.0 / ps, 0.5, 1 - 1.0 / ps, 1 - 0.5 / ps, 1 - 0.2 / ps, 1 - 1e-12, 1.0])
    rays = []
    for i in range(w * h):
        pl = plates[i % len(plates)]
        fwd, right, up = pl[0:3], pl[3:6], pl[6:9]
        uvd = 0.5 / np.tan(np.float32(pl[9]) / np.float32(2))
        u = edge[i % len(edge)] if i % 3 else rng.random()
        v = edge[(i // 7) % len(edge)] if i % 5 else rng.random()
        rays.append(fwd + (u - 0.5) / uvd * right - (v - 0.5) / uvd * up)
    d_rays = torch.from_numpy(np.asarray(rays, np.float32).reshape(h, w, 3)).cuda()
    d_faces = torch.randint(0, 256, (1, 6 * ps * ps), dtype=torch.uint8, device="cuda")
    g = globe(rubix=True)
    out = torch.full((h, w, 4), 7, dtype=torch.uint8, device="cuda")
    fe.warp_rays(d_faces, out, d_rays, None, rowbytes=4 * w, rgba=True, filter="bilinear")
    torch.cuda.synchronize()
    p = br.params(g.fe, w, h, ps, g.grid)
    _, s = br.header_samples(g.lib, p, None, d_rays.cpu().numpy())
    m = s[:, 0] == 1
    assert (s[m, 2] == -1).any() and (s[m, 2] == ps - 1).any() and (s[m, 3] == -1).any() and (s[m, 3] == ps - 1).any()
    pix, _ = g.frame(d_rays.cpu().numpy(), None, d_faces[0], bg.reshape(h, w), 1, ps, table=TABLE)
    assert np.array_equal(out.cpu().numpy(), pix)


# ---- transform forms and batches ---------------------------------------------------------------------------------

def test_per_frame_fields_matrices_and_tables(torch, fe, globe):
    bg = setup(fe, rubix=True)
    g = globe(rubix=True)
    n = 3
    base = field(fe, 2)
    fields = np.stack([base, base[:, ::-1].copy(), np.random.default_rng(12).normal(size=base.shape).astype(np.float32)])
    d_fields = torch.from_numpy(fields).cuda()
    d_faces = faces_for(torch, fe, n)
    tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=1, y0=2, extra=11)
    _, kernel = check(torch, fe, g, 2, bg, d_faces, d_fields, torch.from_numpy(matrices(n)).cuda(), scr, n, False, tables)
    assert "frames/thread=1" in kernel, kernel
    check(torch, fe, g, 2, bg, d_faces, d_fields, None, scr, n, True)
    # one field, one matrix, several frames: the samples are carried from frame to frame
    check(torch, fe, g, 2, bg, d_faces, torch.from_numpy(base).cuda(), torch.from_numpy(matrices(5)[4]).cuda(), scr, n, True, tables)


@pytest.mark.parametrize("form", ["per-frame-matrices", "one-matrix"])
def test_small_view_large_batch_splits_the_frames(torch, fe, globe, form):
    """400 frames of a 96 x 64 view sharing one field, each with its own faces: the frames are split over rows of
    threads"""
    bg = setup(fe)
    g = globe()
    n = 400
    d_rays = torch.from_numpy(field(fe, 1)).cuda()
    distinct = matrices(5)
    d_x = torch.from_numpy(distinct[np.arange(n) % 5] if form == "per-frame-matrices" else distinct[1]).cuda()
    scr = Screens(torch, n, True, x0=3, y0=2, extra=13)
    _, kernel = check(torch, fe, g, 1, bg, faces_for(torch, fe, n), d_rays, d_x, scr, n, form == "one-matrix")
    fpt = int(kernel.split("frames/thread=")[1])
    assert 1 < fpt < n, kernel


@pytest.mark.parametrize("globe_name", ["tetra", "trism", "cube_edge", "cube_corner"])
def test_other_argmax_globes(torch, fe, globe, globe_name):
    bg = setup(fe, globe=globe_name, rubix=True)
    g = globe(globe_name, rubix=True)
    n = 2
    check(torch, fe, g, 2, bg, faces_for(torch, fe, n), torch.from_numpy(field(fe, 2)).cuda(),
          torch.from_numpy(matrices(n, seed=len(globe_name))).cuda(), Screens(torch, n, True, x0=0, y0=0, extra=0), n, False)


@pytest.mark.parametrize("name", ["atlas", "odd"])
def test_face_layouts(torch, fe, globe, name):
    lay = layouts()[name]
    bg = setup(fe, rubix=True, grid=(4, 3.0, 2.0), layout=lay)
    g = globe(rubix=True, grid=(4, 3.0, 2.0))
    n = 2
    d_faces = faces_for(torch, fe, n, lay)
    for k in (1, 3):
        check(torch, fe, g, k, bg, d_faces, torch.from_numpy(field(fe, k)).cuda(), torch.from_numpy(matrices(n)).cuda(),
              Screens(torch, n, True, x0=5, y0=1, extra=7), n, k == 3, layout=lay)


# ---- context state and graphs ------------------------------------------------------------------------------------

def test_the_context_does_not_change(torch, fe):
    setup(fe, rubix=True)
    fe.command("f_lens stereographic")
    fe.build_lensmap(W, H, PS, threads=1)
    state = lambda: (fe.lensmap_packed().tobytes(), fe.display(), fe.build_info, fe.needs_rebuild(W, H, PS), fe.plan_digest(),  # noqa: E731
                     fe.mapped_pixels, fe.width, fe.height, fe.platesize)
    fe.command("f_lens panini")
    d_rays = torch.from_numpy(field(fe, 2)).cuda()
    fe.command("f_lens stereographic")
    before = state()
    out = torch.zeros(2 * W * H * 4, dtype=torch.uint8, device="cuda")
    for k in (1, 2):
        fe.warp_rays(faces_for(torch, fe, 2), out.data_ptr(), d_rays if k == 2 else d_rays[::2, ::2].contiguous(),
                     torch.from_numpy(matrices(2)).cuda(), rowbytes=4 * W, screen_stride=4 * W * H, rgba=True, supersample=k, filter="bilinear")
        torch.cuda.synchronize()
        assert fe.last_kernel.startswith(f"ray_bilinear_kernel<k={k},")
        assert state() == before


@pytest.mark.parametrize("k", [1, 2])
def test_graph_replay_reads_new_matrices_and_tables(torch, fe, globe, k):
    bg = setup(fe, rubix=True)
    g = globe(rubix=True)
    n = 3
    d_faces = faces_for(torch, fe, n)
    d_rays = torch.from_numpy(field(fe, k)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=6, y0=3, extra=5)
    out = scr.new()
    launches = fe.launch_count
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=6, y0=3, rowbytes=scr.rowbytes, nframes=n, rgba=True, tables=tables,
                     screen_stride=scr.stride, supersample=k, filter="bilinear")
    assert fe.launch_count == launches + 1
    d_x.copy_(torch.from_numpy(np.stack([yaw(123.0), yaw(-40.0), yaw(7.0)])))
    tables[1].copy_(torch.from_numpy(np.random.default_rng(9).integers(0, 2**31, 256).astype(np.int32)))
    out.copy_(scr.fill)
    graph.replay()
    torch.cuda.synchronize()
    want = expected(torch, g, scr, k, bg, d_faces, d_rays, d_x, n, False, tables)
    assert torch.equal(out, want), int((out != want).sum())
    del graph
    fe.release_captures()


# ---- refusals ----------------------------------------------------------------------------------------------------

def test_refusals_launch_nothing(bb, torch, fe, palette, cuda_device):
    lib = bb.load_library()
    setup(fe)
    k = 2
    d_rays = torch.from_numpy(field(fe, k)).cuda()
    d_x = torch.from_numpy(matrices(2)).cuda()
    d_faces = faces_for(torch, fe, 2)
    tab = torch.zeros(2 * 256 + 4, dtype=torch.int32, device="cuda")
    out = torch.zeros(2 * W * H * 4 + 16, dtype=torch.uint8, device="cuda")
    R, X, F, O, T = d_rays.data_ptr(), d_x.data_ptr(), d_faces.data_ptr(), out.data_ptr(), tab.data_ptr()

    def call(factor=k, rays=R, rstride=0, xstride=36, o=O, rowbytes=4 * W, tables=None, tstride=0, ctx=None):
        return lib.blinky_warp_device_rays_bilinear(fe._ctx if ctx is None else ctx, F, d_faces.stride(0), rays, rstride, X, xstride, factor, o,
                                                    4 * W * H, rowbytes, 0, 0, 2, 0, tables, tstride, None)

    assert call() == bb.OK and call(factor=1) == bb.OK and call(tables=T, tstride=1024) == bb.OK
    torch.cuda.synchronize()
    launches, kernel = fe.launch_count, fe.last_kernel
    cases = [("factor 5", dict(factor=5)), ("factor 0", dict(factor=0)), ("factor -1", dict(factor=-1)),
             ("ray_stride of a one-sample field", dict(rstride=12 * W * H)), ("ray_stride short by one ray", dict(rstride=12 * k * k * W * H - 12)),
             ("k = 1 ray_stride short by one ray", dict(factor=1, rstride=12 * W * H - 12)),
             ("ray_stride not a multiple of 4", dict(rstride=12 * k * k * W * H + 2)), ("xform_stride short", dict(xstride=32)),
             ("rays misaligned", dict(rays=R + 2)), ("screen misaligned", dict(o=O + 2)), ("rowbytes misaligned", dict(rowbytes=4 * W + 2)),
             ("rowbytes short", dict(rowbytes=4 * W - 4)), ("tables misaligned", dict(tables=T + 4)), ("table_stride", dict(tables=T, tstride=1008)),
             ("NULL rays", dict(rays=None)), ("NULL screen", dict(o=None))]
    for what, kw in cases:
        assert call(**kw) == bb.E_INVALID, what
    assert fe.launch_count == launches and fe.last_kernel == kernel
    fe.command("f_globe fast")
    assert call() == bb.E_STATE and "blinky_set_raymap_device" in lib.blinky_last_error(fe._ctx).decode()
    assert fe.launch_count == launches
    fresh = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        fresh.command("f_globe cube")
        assert call(ctx=fresh._ctx) == bb.E_STATE, "no lensmap installed"
        assert fresh.launch_count == 0
    finally:
        fresh.close()


@pytest.mark.parametrize("k, view", [(1, (65536, 32768)), (4, rr.REFUSED_VIEW)])
def test_31_bit_field_index_is_refused(bb, torch, fe, k, view):
    """k^2 W H = 2^31 samples: refused before anything is launched or written, at k = 1 as at k = 4"""
    w, h = view
    assert k * k * w * h == 2**31
    need = 4 * w * h + w * h + (2 << 30)
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"a {w} x {h} lensmap needs {need} bytes of free device memory; the device reports {free} free of {total}")
    fe.command("f_globe cube")
    fe.set_rgba_table(TABLE)
    fe.set_lensmap(torch.full((h, w), 0x70000000, dtype=torch.int32, device="cuda"), PS, fe.numplates)
    rays = torch.zeros(3 * 1024, dtype=torch.float32, device="cuda")
    out = torch.full((4096,), 77, dtype=torch.uint8, device="cuda")
    d_faces = torch.zeros(6 * PS * PS, dtype=torch.uint8, device="cuda")
    lib = bb.load_library()
    launches, last = fe.launch_count, fe.last_kernel
    rc = lib.blinky_warp_device_rays_bilinear(fe._ctx, d_faces.data_ptr(), 0, rays.data_ptr(), 0, None, 0, k, out.data_ptr(), 0, 4 * w, 0, 0, 1,
                                              0, None, 0, None)
    err = lib.blinky_last_error(fe._ctx).decode()
    assert rc == bb.E_INVALID and "31-bit" in err and str(2**31) in err, err
    assert fe.launch_count == launches and fe.last_kernel == last
    torch.cuda.synchronize()
    assert bool((out == 77).all())
