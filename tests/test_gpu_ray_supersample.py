"""The supersampled warp from a ray field (blinky_warp_device_rays_supersampled, warp_rays(supersample=k)) on the GPU.
The oracle: frame f is the k x k box average, with round-half-up per byte, of blinky_warp_device_rays_rgba at k*W x k*H
whose background is the W x H background with each byte repeated k x k.  The same context installs an all-unmapped
k*W x k*H lensmap of the same plate size (the ray warps read only its size, plate size and background), warps, averages
on the GPU, then reinstalls the W x H map and background and runs the new call.  With keep_unmapped a pixel is left
alone exactly when none of its samples is mapped, found as the pixels of two keep_unmapped warps into different
sentinels that differ.  Every byte of each output buffer is compared, the bytes outside the view included."""
import numpy as np
import pytest

import ray_reference as rr
from test_gpu_ray_warp import Screens, layouts, matrices, yaw

pytestmark = pytest.mark.gpu

W, H, PS = 96, 64, 48
TABLE = np.random.default_rng(2).integers(0, 2**32, 256, dtype=np.uint32)


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture()
def fe(bb, palette, cuda_device):
    c = bb.Fisheye(device=cuda_device, palette=palette)
    yield c
    c.close()


def install(fe, w, h, bg, ps=PS):
    """an all-unmapped w x h lensmap of plate size ps, and its background"""
    fe.set_lensmap(np.full((h, w), 0x70000000, np.uint32), ps, fe.numplates)
    fe.set_background(np.ascontiguousarray(bg).reshape(-1))


def setup(fe, globe="cube", rubix=False, grid=None, layout=None, seed=3):
    """fe on globe / panini at f_fov 180 with a W x H map installed; the background"""
    if grid:
        fe.set_rubixgrid(*grid)
    fe.command(f"f_globe {globe}")
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    fe.set_rubix(rubix)
    fe.set_rgba_table(TABLE)
    bg = np.random.default_rng(seed).integers(0, 256, W * H, dtype=np.uint8)
    install(fe, W, H, bg)
    if layout:
        fe.set_face_layout(*layout)
    return bg


def field(fe, k, seed=7):
    """the exported panini field at k*W x k*H with some pixels wholly unmapped (zero rays), some partly, and some
    random and non-finite rays"""
    rays = fe.raymap(k * W, k * H)
    blocks = rays.reshape(H, k, W, k, 3)
    blocks[::7, :, ::5] = 0
    blocks[3::11, 0, 2::9, k - 1] = 0
    blocks[5::13, k - 1, 1::7, :] = 0
    r = rays.reshape(-1, 3)
    r[::53] = np.random.default_rng(seed).normal(size=r[::53].shape).astype(np.float32)
    r[9::307] = [np.inf, 0, 1]
    return rays


def faces_for(torch, fe, n, layout=None, seed=1, ps=PS):
    rng = np.random.default_rng(seed)
    if layout is None:
        return torch.from_numpy(rng.integers(0, 256, (n, fe.numplates * ps * ps), dtype=np.uint8)).cuda()
    rowbytes, origins = layout
    rows = max(y for _, y in origins) + ps
    return torch.from_numpy(rng.integers(0, 256, (n, rows, rowbytes), dtype=np.uint8)).cuda()


def oracle(torch, fe, k, bg, d_faces, d_rays, d_x, n, keep, tables=None, w=W, h=H, ps=PS):
    """(the [n, h, w, 4] box averages, the [n, h, w] pixels with a mapped sample or None) by the one-sample warp at k*w x
    k*h; fe is left with the w x h map and background installed again"""
    kw, kh = k * w, k * h
    install(fe, kw, kh, np.repeat(np.repeat(bg.reshape(h, w), k, 0), k, 1), ps)

    def big(keep_big, fill):
        out = torch.full((n, kh, kw, 4), fill, dtype=torch.uint8, device="cuda")
        fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, rowbytes=4 * kw, screen_stride=4 * kw * kh, nframes=n, keep_unmapped=keep_big,
                     rgba=True, tables=tables)
        assert fe.last_kernel.startswith("ray_warp_kernel<"), fe.last_kernel
        return out

    s = big(False, 0).view(n, h, k, w, k, 4).to(torch.int32).sum((2, 4))
    avg = ((s + k * k // 2) // (k * k)).to(torch.uint8)
    mapped = None
    if keep:
        a, b = big(True, 0), big(True, 255)
        mapped = (a != b).any(-1).logical_not().view(n, h, k, w, k).any(4).any(2)
    install(fe, w, h, bg, ps)
    torch.cuda.synchronize()
    return avg, mapped


def expected(scr, avg, mapped, n, w=W, h=H):
    """the screens scr.fill with the view rectangles of n frames written by the rule"""
    exp = scr.fill.clone()
    for f in range(n):
        v = exp.as_strided((h, w, 4), (scr.rowbytes, 4, 1), f * scr.stride + scr.y0 * scr.rowbytes + 4 * scr.x0)
        v.copy_(avg[f] if mapped is None else avg[f].where(mapped[f][..., None], v))
    return exp


def run(torch, fe, k, d_faces, d_rays, d_x, scr, n, keep, tables=None):
    out = scr.new()
    launches = fe.launch_count
    fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=scr.x0, y0=scr.y0, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep, rgba=True,
                 tables=tables, screen_stride=scr.stride, supersample=k)
    torch.cuda.synchronize()
    assert fe.launch_count == launches + 1
    return out, fe.last_kernel


def by_reference(torch, host, k, bg, d_faces, d_rays, d_x, n, keep, tables=None, w=W, h=H, ps=PS, band=None):
    """(avg, mapped) as oracle() gives them, by tests/ray_reference.py (no project kernel); host: its HostGlobe on the
    globe, rubix state and grid of fe.  band: output rows at a time (the 4K fields)"""
    faces, field = d_faces.cpu().numpy(), d_rays.cpu().numpy()
    xs = None if d_x is None else d_x.cpu().numpy()
    tabs = None if tables is None else tables.cpu().numpy().view(np.uint32)
    band = band or h
    avg = np.empty((n, h, w, 4), np.uint8)
    mapped = np.empty((n, h, w), bool)
    for f in range(n):
        fld = field if field.ndim == 3 else field[f]
        M = None if xs is None else (xs if xs.ndim == 2 else xs[f])
        tab = TABLE if tabs is None else (tabs if tabs.ndim == 1 else tabs[f])
        for y in range(0, h, band):
            avg[f, y:y + band], mapped[f, y:y + band] = rr.frame(host, fld[k * y:k * (y + band)], M, faces[min(f, len(faces) - 1)],
                                                                 bg.reshape(h, w)[y:y + band], k, ps, table=tab)
    return torch.from_numpy(avg).cuda(), torch.from_numpy(mapped).cuda() if keep else None


def check(torch, fe, k, bg, d_faces, d_rays, d_x, scr, n, keep, tables=None, expect_kernel=None, host=None):
    """the new call against the oracle (and, given host, tests/ray_reference.py), every byte of the screens; the
    kernel's description"""
    got, kernel = run(torch, fe, k, d_faces, d_rays, d_x, scr, n, keep, tables)
    if expect_kernel:
        assert kernel.startswith(expect_kernel), kernel
    avg, mapped = oracle(torch, fe, k, bg, d_faces, d_rays, d_x, n, keep, tables)
    if keep:
        assert bool(mapped.any()) and not bool(mapped.all()), "some pixels wholly unmapped, some not"
    want = expected(scr, avg, mapped, n)
    bad = (got != want).nonzero().flatten()
    assert bad.numel() == 0, (kernel, bad.numel(), bad[:8].tolist())
    if host is not None:
        want = expected(scr, *by_reference(torch, host, k, bg, d_faces, d_rays, d_x, n, keep, tables), n)
        bad = (got != want).nonzero().flatten()
        assert bad.numel() == 0, ("ray_reference", kernel, bad.numel(), bad[:8].tolist())
    return kernel


# ---- every kernel instance against the rule ----------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["context", "frames", "shared"])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("rubix", [False, True])
@pytest.mark.parametrize("k", [2, 3, 4])
def test_every_instance_follows_the_rule(bb, palette, torch, fe, k, rubix, keep, mode):
    bg = setup(fe, rubix=rubix)
    host = rr.HostGlobe(bb, palette, "cube", rubix=rubix)
    n = 3
    d_rays = torch.from_numpy(field(fe, k)).cuda()
    d_x = torch.from_numpy(np.stack([yaw(0), yaw(29), yaw(-71)])).cuda()
    tables = None
    if mode == "frames":
        tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    elif mode == "shared":
        tables = torch.from_numpy(np.random.default_rng(8).integers(0, 2**31, 256).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=3, y0=5, extra=13)
    tag = f"ray_supersample_kernel<k={k},rubix={int(rubix)},keep={int(keep)},tables={int(mode == 'frames')}>"
    try:
        check(torch, fe, k, bg, faces_for(torch, fe, n), d_rays, d_x, scr, n, keep, tables, expect_kernel=tag, host=host)
    finally:
        host.close()


@pytest.mark.parametrize("keep", [False, True])
def test_repeated_rays_equal_the_one_sample_warp(bb, torch, fe, keep):
    """a field whose k x k samples of a pixel are all that pixel's ray gives blinky_warp_device_rays_rgba's output"""
    setup(fe, rubix=True)
    rays = field(fe, 1)
    n = 3
    d_faces = faces_for(torch, fe, n)
    d_x = torch.from_numpy(matrices(n)).cuda()
    scr = Screens(torch, n, True, x0=4, y0=1, extra=12)
    one = scr.new()
    fe.warp_rays(d_faces, one.data_ptr(), torch.from_numpy(rays).cuda(), d_x, x0=4, y0=1, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep,
                 rgba=True, screen_stride=scr.stride)
    torch.cuda.synchronize()
    for k in (2, 3, 4):
        rep = torch.from_numpy(np.ascontiguousarray(np.repeat(np.repeat(rays, k, 0), k, 1))).cuda()
        got, kernel = run(torch, fe, k, d_faces, rep, d_x, scr, n, keep)
        assert torch.equal(got, one), (kernel, int((got != one).sum()))


# ---- transform forms ---------------------------------------------------------------------------------------------

def test_per_frame_fields_one_matrix_and_no_matrix(bb, torch, fe):
    bg = setup(fe, rubix=True)
    n = 3
    base = field(fe, 2)
    rng = np.random.default_rng(12)
    fields = np.stack([base, base[:, ::-1].copy(), rng.normal(size=base.shape).astype(np.float32)])
    d_fields = torch.from_numpy(fields).cuda()
    d_faces = faces_for(torch, fe, n)
    scr = Screens(torch, n, True, x0=1, y0=2, extra=11)
    kernel = check(torch, fe, 2, bg, d_faces, d_fields, torch.from_numpy(matrices(5)[3]).cuda(), scr, n, False)
    assert "frames/thread=1" in kernel, kernel
    check(torch, fe, 2, bg, d_faces, d_fields, None, scr, n, True)
    # one field, one matrix, several frames: the texels are carried from frame to frame
    d_base = torch.from_numpy(base).cuda()
    check(torch, fe, 2, bg, d_faces, d_base, torch.from_numpy(matrices(5)[4]).cuda(), scr, n, True)
    check(torch, fe, 2, bg, d_faces, d_base, None, scr, n, False)


@pytest.mark.parametrize("form", ["per-frame-matrices", "one-matrix"])
def test_small_view_large_batch_splits_the_frames(bb, torch, fe, form):
    """400 frames of a 96 x 64 view sharing one field: the frames are split over rows of threads.  Each frame has its
    own faces (the warp and the oracle step through them by the dense frame size)."""
    bg = setup(fe)
    n = 400
    d_rays = torch.from_numpy(field(fe, 3)).cuda()
    distinct = matrices(5)
    d_x = torch.from_numpy(distinct[np.arange(n) % 5] if form == "per-frame-matrices" else distinct[1]).cuda()
    scr = Screens(torch, n, True, x0=3, y0=2, extra=13)
    kernel = check(torch, fe, 3, bg, faces_for(torch, fe, n), d_rays, d_x, scr, n, form == "one-matrix")
    fpt = int(kernel.split("frames/thread=")[1])
    assert 1 < fpt < n, kernel


# ---- face layouts and globes -------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["atlas", "padded", "odd"])
def test_face_layouts(bb, torch, fe, name):
    lay = layouts()[name]
    bg = setup(fe, rubix=True, grid=(4, 3.0, 2.0), layout=lay)
    n = 3
    d_faces = faces_for(torch, fe, n, lay)
    for k in (2, 4):
        check(torch, fe, k, bg, d_faces, torch.from_numpy(field(fe, k)).cuda(), torch.from_numpy(matrices(n)).cuda(),
              Screens(torch, n, True, x0=5, y0=1, extra=7), n, k == 4, expect_kernel=f"ray_supersample_kernel<k={k},rubix=1")


@pytest.mark.parametrize("globe", ["tetra", "trism", "cube_edge"])
def test_other_argmax_globes(bb, torch, fe, globe):
    bg = setup(fe, globe=globe, rubix=True)
    n = 3
    check(torch, fe, 3, bg, faces_for(torch, fe, n), torch.from_numpy(field(fe, 3)).cuda(), torch.from_numpy(matrices(n, seed=len(globe))).cuda(),
          Screens(torch, n, True, x0=0, y0=0, extra=0), n, False)


# ---- context state and graphs ------------------------------------------------------------------------------------

def test_the_context_does_not_change(bb, torch, fe):
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
    fe.warp_rays(faces_for(torch, fe, 2), out.data_ptr(), d_rays, torch.from_numpy(matrices(2)).cuda(), rowbytes=4 * W, screen_stride=4 * W * H,
                 rgba=True, supersample=2)
    torch.cuda.synchronize()
    assert fe.last_kernel.startswith("ray_supersample_kernel<k=2,")
    assert state() == before


def test_graph_replay_reads_new_matrices_and_tables(bb, torch, fe):
    bg = setup(fe, rubix=True)
    n = 3
    d_faces = faces_for(torch, fe, n)
    d_rays = torch.from_numpy(field(fe, 2)).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    scr = Screens(torch, n, True, x0=6, y0=3, extra=5)
    out = scr.new()
    launches = fe.launch_count
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=6, y0=3, rowbytes=scr.rowbytes, nframes=n, rgba=True, tables=tables,
                     screen_stride=scr.stride, supersample=2)
    assert fe.launch_count == launches + 1
    # new matrices and a new table for frame 1, written in stream order before the replay
    d_x.copy_(torch.from_numpy(np.stack([yaw(123.0), yaw(-40.0), yaw(7.0)])))
    tables[1].copy_(torch.from_numpy(np.random.default_rng(9).integers(0, 2**31, 256).astype(np.int32)))
    out.copy_(scr.fill)
    g.replay()
    torch.cuda.synchronize()
    avg, _ = oracle(torch, fe, 2, bg, d_faces, d_rays, d_x, n, False, tables)
    want = expected(scr, avg, None, n)
    assert torch.equal(out, want), int((out != want).sum())
    del g
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

    def call(factor=k, rays=R, rstride=0, o=O, rowbytes=4 * W, tables=None, tstride=0, ctx=None):
        return lib.blinky_warp_device_rays_supersampled(fe._ctx if ctx is None else ctx, F, d_faces.stride(0), rays, rstride, X, 36, factor, o,
                                                        4 * W * H, rowbytes, 0, 0, 2, 0, tables, tstride, None)

    assert call() == bb.OK and call(tables=T, tstride=1024) == bb.OK
    torch.cuda.synchronize()
    launches, kernel = fe.launch_count, fe.last_kernel
    cases = [("factor 1", dict(factor=1)), ("factor 5", dict(factor=5)), ("factor 0", dict(factor=0)),
             ("ray_stride of a one-sample field", dict(rstride=12 * W * H)), ("ray_stride short by one ray", dict(rstride=12 * k * k * W * H - 12)),
             ("ray_stride not a multiple of 4", dict(rstride=12 * k * k * W * H + 2)), ("rays misaligned", dict(rays=R + 2)),
             ("screen misaligned", dict(o=O + 2)), ("rowbytes misaligned", dict(rowbytes=4 * W + 2)), ("tables misaligned", dict(tables=T + 4)),
             ("table_stride", dict(tables=T, tstride=1008)), ("NULL rays", dict(rays=None)), ("NULL screen", dict(o=None))]
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


# ---- 4K ----------------------------------------------------------------------------------------------------------

def test_4k_look_around_at_k2(bb, palette, torch, fe):
    """a 3-frame 4K look-around from the exported panini field at 7680 x 4320 (~400 MB)"""
    W4, H4, P4, k, n = 3840, 2160, 2048, 2, 3
    fe.command("f_globe cube")
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    fe.set_rgba_table(TABLE)
    bg = np.random.default_rng(5).integers(0, 256, W4 * H4, dtype=np.uint8)
    install(fe, W4, H4, bg, P4)
    d_rays = torch.empty((k * H4, k * W4, 3), dtype=torch.float32, device="cuda")
    fe.raymap(k * W4, k * H4, out=d_rays)
    d_x = torch.from_numpy(np.stack([yaw(0), yaw(33), yaw(-120)])).cuda()
    d_faces = torch.randint(0, 256, (n, 6 * P4 * P4), dtype=torch.uint8, device="cuda")
    out = torch.full((n, H4, W4, 4), 77, dtype=torch.uint8, device="cuda")
    fe.warp_rays(d_faces, out, d_rays, d_x, rowbytes=4 * W4, screen_stride=4 * W4 * H4, rgba=True, supersample=k)
    torch.cuda.synchronize()
    assert fe.last_kernel.startswith("ray_supersample_kernel<k=2,rubix=0,keep=0,tables=0>"), fe.last_kernel
    avg, _ = oracle(torch, fe, k, bg, d_faces, d_rays, d_x, n, False, w=W4, h=H4, ps=P4)
    assert torch.equal(out, avg), int((out != avg).any(-1).sum())
    host = rr.HostGlobe(bb, palette, "cube")
    try:
        avg, _ = by_reference(torch, host, k, bg, d_faces, d_rays, d_x, n, False, w=W4, h=H4, ps=P4, band=270)
    finally:
        host.close()
    assert torch.equal(out, avg), ("ray_reference", int((out != avg).any(-1).sum()))
