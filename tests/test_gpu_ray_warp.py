"""The warp from a ray field turned by a per-frame matrix (blinky_warp_device_rays[_rgba]) on the GPU.  The rule: frame f
equals blinky_set_raymap of the field turned in numpy float32 by M_f, followed by a one-frame blinky_warp_device_view of
that frame, on a second context with the same globe, palette, background, rubix state and face layout.  Every byte of
each output buffer is compared, the bytes outside the view included.  Covered: every kernel instance, face layouts,
the transform forms, CUDA graphs, refusals, a 4K look-around, adversarial rays and matrices on every argmax globe, the
exported fields of extreme zooms, and the largest plate size a ray map takes."""
import numpy as np
import pytest

from conftest import ALL_LENSES
from test_raymap_host_only import adversarial_rays, u_one_rays

pytestmark = pytest.mark.gpu

W, H, PS = 96, 64, 48


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture()
def pair(bb, palette, cuda_device):
    """(the context that warps from rays, the one that installs each turned field as a ray map)"""
    a = bb.Fisheye(device=cuda_device, palette=palette)
    b = bb.Fisheye(device=cuda_device, palette=palette)
    yield a, b
    a.close()
    b.close()


def turned(rays, M):
    """numpy's float32 (M[k,0]*x + M[k,1]*y) + M[k,2]*z: the turn the warp must repeat"""
    M = np.asarray(M, np.float32)
    x, y, z = rays[..., 0], rays[..., 1], rays[..., 2]
    with np.errstate(all="ignore"):
        return np.stack([(M[k, 0] * x + M[k, 1] * y) + M[k, 2] * z for k in range(3)], axis=-1).astype(np.float32)


def yaw(deg):
    a = np.radians(deg)
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32)


def matrices(n, seed=5):
    """yaws, roll plus pitch, non-orthogonal, the identity"""
    rng = np.random.default_rng(seed)
    out = [yaw(17.0 * i) for i in range(max(1, n - 3))]
    a, b = np.radians(23.0), np.radians(-31.0)
    roll = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], np.float32)
    pitch = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]], np.float32)
    out += [(roll @ pitch).astype(np.float32), (np.eye(3) + 0.3 * rng.normal(size=(3, 3))).astype(np.float32), np.eye(3, dtype=np.float32)]
    return np.stack(out[:n]).astype(np.float32)


def setup(pair, globe="cube", lens="panini", rubix=False, grid=None, layout=None, bg_seed=3):
    """both contexts on globe / lens at W x H x PS, same background, rubix state and face layout; the lens's rays"""
    rng = np.random.default_rng(bg_seed)
    bg = rng.integers(0, 256, W * H, dtype=np.uint8)
    for fe in pair:
        if grid:
            fe.set_rubixgrid(*grid)
        fe.command(f"f_globe {globe}")
        fe.command(f"f_lens {lens}")
        fe.command("f_fov 180")
        fe.set_rubix(rubix)
        fe.build_lensmap(W, H, PS, threads=1)
        fe.set_background(bg)
        if layout:
            fe.set_face_layout(*layout)
    rays = pair[0].raymap(W, H)
    # some pixels off the lens: random, zero and non-finite rays
    r = rays.reshape(-1, 3)
    r[::53] = np.random.default_rng(7).normal(size=r[::53].shape).astype(np.float32)
    r[5::211] = 0
    r[9::307] = [np.inf, 0, 1]
    return rays


def faces_for(torch, fe, nframes, layout=None, seed=1):
    """device faces of nframes frames: dense [N, numplates*ps*ps] or the layout's [N, rows, rowbytes] surfaces"""
    rng = np.random.default_rng(seed)
    if layout is None:
        return torch.from_numpy(rng.integers(0, 256, (nframes, fe.numplates * PS * PS), dtype=np.uint8)).cuda()
    rowbytes, origins = layout
    rows = max(y for _, y in origins) + PS
    return torch.from_numpy(rng.integers(0, 256, (nframes, rows, rowbytes), dtype=np.uint8)).cuda()


class Screens:
    """nframes screens holding seeded bytes, a view rectangle at (x0, y0)"""

    def __init__(self, torch, nframes, rgba, x0, y0, extra=13, seed=9):
        self.bpp = 4 if rgba else 1
        self.x0, self.y0 = x0, y0
        self.rowbytes = (x0 + W + extra) * self.bpp
        self.stride = (y0 + H + 3) * self.rowbytes + 4 * self.bpp
        g = torch.Generator().manual_seed(seed)
        self.fill = torch.randint(0, 256, (nframes * self.stride,), dtype=torch.uint8, generator=g).cuda()

    def new(self):
        return self.fill.clone()


def reference(torch, ref, rays_f, M_f, d_faces_f, scr, f, keep, rgba, table_f):
    """frame f by the rule: set_raymap of the turned field (host path), one-frame warp_view into frame f's bytes"""
    t = rays_f if M_f is None else turned(rays_f, M_f)
    with np.errstate(all="ignore"):
        ref.set_raymap(np.ascontiguousarray(t), PS)
    out = scr.fill[f * scr.stride:(f + 1) * scr.stride].clone()
    ref.warp_view(d_faces_f, out.data_ptr(), x0=scr.x0, y0=scr.y0, rowbytes=scr.rowbytes, nframes=1, keep_unmapped=keep, rgba=rgba,
                  screen_stride=scr.stride, tables=table_f)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def check_batch(torch, fe, ref, rays, xs, d_faces, scr, keep, rgba, tables=None, per_frame_rays=None, expect_kernel=None):
    """warp_rays of len(xs) frames (xs None: no turn) against the rule, frame by frame"""
    n = len(xs) if xs is not None else (len(per_frame_rays) if per_frame_rays is not None else 1)
    out = scr.new()
    d_rays = torch.from_numpy(per_frame_rays if per_frame_rays is not None else rays).cuda()
    d_x = None if xs is None else torch.from_numpy(xs).cuda()
    launches = fe.launch_count
    fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=scr.x0, y0=scr.y0, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep, rgba=rgba,
                 tables=tables, screen_stride=scr.stride)
    torch.cuda.synchronize()
    assert fe.launch_count == launches + 1
    kernel = fe.last_kernel
    if expect_kernel:
        assert kernel.startswith(expect_kernel), kernel
    got = out.cpu().numpy()
    for f in range(n):
        rf = per_frame_rays[f] if per_frame_rays is not None else rays
        table_f = None if tables is None else (tables if tables.dim() == 1 else tables[f])
        want = reference(torch, ref, rf, None if xs is None else xs[f], d_faces[f:f + 1], scr, f, keep, rgba, table_f)
        have = got[f * scr.stride:(f + 1) * scr.stride]
        bad = np.nonzero(have != want)[0]
        assert bad.size == 0, (kernel, f, bad.size, bad[:8].tolist())
    # the untouched tail past the last frame
    assert np.array_equal(got[n * scr.stride:], scr.fill.cpu().numpy()[n * scr.stride:])
    return kernel


# ---- every kernel instance against the rule ----------------------------------------------------------------------

@pytest.mark.parametrize("quad", [True, False])
@pytest.mark.parametrize("mode", ["8bit", "rgba", "tables"])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("rubix", [False, True])
def test_every_instance_follows_the_rule(bb, torch, pair, quad, mode, keep, rubix):
    fe, ref = pair
    rays = setup(pair, rubix=rubix)
    rgba = mode != "8bit"
    n = 5
    xs = matrices(n)
    table = np.random.default_rng(2).integers(0, 2**32, 256, dtype=np.uint32)
    for c in pair:
        c.set_rgba_table(table)
    tables = None
    if mode == "tables":
        tables = torch.from_numpy(np.random.default_rng(4).integers(0, 2**31, (n, 256)).astype(np.int32)).cuda()
    # quads: origin, pitch and frame stride on 4-pixel words; otherwise an odd origin
    scr = Screens(torch, n, rgba, x0=8 if quad else 3, y0=2, extra=12 if quad else 13)
    if quad:
        assert scr.rowbytes % (4 * scr.bpp) == 0 and scr.stride % (4 * scr.bpp) == 0
    d_faces = faces_for(torch, fe, n)
    tag = f"ray_warp_kernel<quad={int(quad)},rubix={int(rubix)},rgba={int(rgba)},keep={int(keep)},tables={int(mode == 'tables')}>"
    check_batch(torch, fe, ref, rays, xs, d_faces, scr, keep, rgba, tables=tables, expect_kernel=tag)


def test_shared_tables_and_odd_pitch(bb, torch, pair):
    """one table for every frame (stride 0: the RGBA instance without per-frame tables), an odd pitch in 8-bit"""
    fe, ref = pair
    rays = setup(pair, rubix=True)
    xs = matrices(3)
    d_faces = faces_for(torch, fe, 3)
    tab = torch.from_numpy(np.random.default_rng(8).integers(0, 2**31, 256).astype(np.int32)).cuda()
    check_batch(torch, fe, ref, rays, xs, d_faces, Screens(torch, 3, True, 4, 1, extra=12), False, True, tables=tab,
                expect_kernel="ray_warp_kernel<quad=1,rubix=1,rgba=1,keep=0,tables=0>")
    check_batch(torch, fe, ref, rays, xs, d_faces, Screens(torch, 3, False, 4, 1, extra=11), True, False,
                expect_kernel="ray_warp_kernel<quad=0,")


# ---- face layouts ------------------------------------------------------------------------------------------------

def layouts():
    ps = PS
    atlas = (3 * ps, [(0, 0), (ps, 0), (2 * ps, 0), (0, ps), (ps, ps), (2 * ps, ps)])
    padded = (ps + 40, [(16, i * (ps + 3)) for i in range(6)])
    odd = (2 * ps + 37, [(5 + (i % 2) * (ps + 7), 3 + (i // 2) * (ps + 1)) for i in range(6)])
    return {"atlas": atlas, "padded": padded, "odd": odd}


@pytest.mark.parametrize("name", ["atlas", "padded", "odd"])
@pytest.mark.parametrize("rubix", [False, True])
def test_face_layouts(bb, torch, pair, name, rubix):
    fe, ref = pair
    lay = layouts()[name]
    rays = setup(pair, rubix=rubix, grid=(4, 3.0, 2.0) if rubix else None, layout=lay)
    xs = matrices(4)
    d_faces = faces_for(torch, fe, 4, lay)
    for quad in (True, False):
        scr = Screens(torch, 4, False, 8 if quad else 1, 1, extra=12 if quad else 13)
        check_batch(torch, fe, ref, rays, xs, d_faces, scr, quad, False, expect_kernel=f"ray_warp_kernel<quad={int(quad)}")


@pytest.mark.parametrize("globe", ["tetra", "trism", "cube_edge"])
def test_other_argmax_globes(bb, torch, pair, globe):
    fe, ref = pair
    rays = setup(pair, globe=globe, rubix=True)
    xs = matrices(4, seed=globe.__len__())
    d_faces = faces_for(torch, fe, 4)
    check_batch(torch, fe, ref, rays, xs, d_faces, Screens(torch, 4, True, 0, 0, extra=0), False, True)


# ---- transform forms ---------------------------------------------------------------------------------------------

def test_per_frame_fields_and_one_shared_matrix(bb, torch, pair):
    fe, ref = pair
    rays = setup(pair, rubix=True)
    n = 3
    rng = np.random.default_rng(12)
    fields = np.stack([rays, turned(rays, yaw(40)), rng.normal(size=rays.shape).astype(np.float32)])
    d_faces = faces_for(torch, fe, n)
    scr = Screens(torch, n, False, 4, 2, extra=12)
    # ray_stride != 0, one matrix (xform_stride 0)
    out = scr.new()
    M = matrices(5)[3]
    fe.warp_rays(d_faces, out.data_ptr(), torch.from_numpy(fields).cuda(), torch.from_numpy(M).cuda(), x0=4, y0=2, rowbytes=scr.rowbytes,
                 nframes=n, screen_stride=scr.stride)
    torch.cuda.synchronize()
    assert "frames/thread=1" in fe.last_kernel
    got = out.cpu().numpy()
    for f in range(n):
        want = reference(torch, ref, fields[f], M, d_faces[f:f + 1], scr, f, False, False, None)
        assert np.array_equal(got[f * scr.stride:(f + 1) * scr.stride], want), f
    # per-frame fields, no turn
    check_batch(torch, fe, ref, rays, None, d_faces, scr, False, False, per_frame_rays=fields)


def test_null_and_identity_for_every_inverse_lens(bb, torch, pair):
    """xforms None equals the untransformed set_raymap warp; the identity equals None for the exported rays of every
    inverse lens (a turn by the identity changes only the sign of a zero or turns an infinite component into NaN)"""
    fe, ref = pair
    setup(pair)
    d_faces = faces_for(torch, fe, 1)
    scr = Screens(torch, 1, False, 0, 0, extra=0)
    eye = torch.eye(3, dtype=torch.float32).cuda()
    checked = 0
    for lens in ALL_LENSES:
        for c in pair:
            c.command(f"f_lens {lens}")
        try:
            rays = fe.raymap(W, H)
        except bb.BlinkyError:
            continue   # forward-only lens, or a zoom it cannot do
        d_rays = torch.from_numpy(rays).cuda()
        a, b = scr.new(), scr.new()
        fe.warp_rays(d_faces, a.data_ptr(), d_rays, None, rowbytes=W, screen_stride=scr.stride)
        fe.warp_rays(d_faces, b.data_ptr(), d_rays, eye, rowbytes=W, screen_stride=scr.stride)
        torch.cuda.synchronize()
        want = reference(torch, ref, rays, None, d_faces[0:1], scr, 0, False, False, None)
        assert np.array_equal(a.cpu().numpy(), want), lens
        assert np.array_equal(b.cpu().numpy(), want), lens
        checked += 1
    assert checked >= 15, checked


# ---- context state -----------------------------------------------------------------------------------------------

def test_the_context_does_not_change(bb, torch, pair):
    fe, _ = pair
    rays = setup(pair, rubix=True)
    before = (fe.lensmap_packed().copy(), fe.display(), fe.build_info, fe.needs_rebuild(W, H, PS), fe.plan_digest(), fe.mapped_pixels)
    d_faces = faces_for(torch, fe, 2)
    out = torch.zeros(2 * W * H, dtype=torch.uint8).cuda()
    fe.warp_rays(d_faces, out.data_ptr(), torch.from_numpy(rays).cuda(), torch.from_numpy(matrices(2)).cuda(), rowbytes=W, screen_stride=W * H)
    torch.cuda.synchronize()
    after = (fe.lensmap_packed(), fe.display(), fe.build_info, fe.needs_rebuild(W, H, PS), fe.plan_digest(), fe.mapped_pixels)
    assert np.array_equal(before[0], after[0]) and before[1:] == after[1:]


# ---- CUDA graphs -------------------------------------------------------------------------------------------------

def test_graph_replay_reads_new_matrices_and_keeps_its_state(bb, torch, pair):
    fe, ref = pair
    rays = setup(pair, rubix=True)
    n = 4
    d_faces = faces_for(torch, fe, n)
    scr = Screens(torch, n, False, 8, 2, extra=12)
    d_rays = torch.from_numpy(rays).cuda()
    d_x = torch.from_numpy(matrices(n)).cuda()
    out = scr.new()
    launches = fe.launch_count
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp_rays(d_faces, out.data_ptr(), d_rays, d_x, x0=8, y0=2, rowbytes=scr.rowbytes, nframes=n, screen_stride=scr.stride)
        with pytest.raises(bb.BlinkyError) as e:
            fe.release_captures()
        assert e.value.code == bb.E_INVALID
    assert fe.launch_count == launches + 1
    new_x = matrices(n, seed=99)[::-1].copy()
    new_x[0] = yaw(123.0)
    d_x.copy_(torch.from_numpy(new_x))
    out.copy_(scr.fill)
    g.replay()
    torch.cuda.synchronize()
    replayed = out.cpu().numpy()
    eager = scr.new()
    fe.warp_rays(d_faces, eager.data_ptr(), d_rays, d_x, x0=8, y0=2, rowbytes=scr.rowbytes, nframes=n, screen_stride=scr.stride)
    torch.cuda.synchronize()
    assert np.array_equal(replayed, eager.cpu().numpy())
    for f in (0, n - 1):
        want = reference(torch, ref, rays, new_x[f], d_faces[f:f + 1], scr, f, False, False, None)
        assert np.array_equal(replayed[f * scr.stride:(f + 1) * scr.stride], want), f
    # a rebuild to another lens (same view size) and another globe: the replay still renders the capture's state
    fe.command("f_lens stereographic")
    fe.build_lensmap(W, H, PS, threads=1)
    fe.command("f_globe trism")
    out.copy_(scr.fill)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), replayed)
    del g
    fe.release_captures()


# ---- refusals ----------------------------------------------------------------------------------------------------

def test_refusals_launch_nothing(bb, torch, pair, palette, cuda_device):
    fe, _ = pair
    lib = bb.load_library()
    rays = setup(pair)
    d_rays = torch.from_numpy(rays).cuda()
    d_x = torch.from_numpy(matrices(2)).cuda()
    d_faces = faces_for(torch, fe, 2)
    out = torch.zeros(2 * W * H * 4, dtype=torch.uint8).cuda()
    R, X, F, O = d_rays.data_ptr(), d_x.data_ptr(), d_faces.data_ptr(), out.data_ptr()
    fs = d_faces.stride(0)

    def call(faces=F, fstride=fs, rays=R, rstride=0, xf=X, xstride=36, o=O, ostride=W * H, rowbytes=W, x0=0, y0=0, n=2, rgba=False,
             tables=None, tstride=0, ctx=None):
        c = fe._ctx if ctx is None else ctx
        if rgba:
            return lib.blinky_warp_device_rays_rgba(c, faces, fstride, rays, rstride, xf, xstride, o, ostride, rowbytes, x0, y0, n, 0, tables,
                                                    tstride, None)
        return lib.blinky_warp_device_rays(c, faces, fstride, rays, rstride, xf, xstride, o, ostride, rowbytes, x0, y0, n, 0, None)

    assert call() == bb.OK
    torch.cuda.synchronize()
    launches, kernel = fe.launch_count, fe.last_kernel
    cases = [("NULL faces", dict(faces=None)), ("NULL rays", dict(rays=None)), ("NULL screen", dict(o=None)),
             ("rays misaligned", dict(rays=R + 2)), ("xforms misaligned", dict(xf=X + 2)),
             ("ray_stride too small", dict(rstride=12 * W * H - 4)), ("ray_stride not a multiple of 4", dict(rstride=12 * W * H + 2)),
             ("xform_stride too small", dict(xstride=32)), ("xform_stride not a multiple of 4", dict(xstride=38)),
             ("65536 frames", dict(n=65536, ostride=0)), ("rowbytes", dict(rowbytes=W - 1)), ("negative origin", dict(x0=-1)),
             ("frame stride", dict(ostride=W * H - 1)), ("RGBA pitch", dict(rgba=True, rowbytes=4 * W + 2, ostride=8 * W * H)),
             ("tables misaligned", dict(rgba=True, rowbytes=4 * W, ostride=4 * W * H, tables=X + 4)),
             ("table_stride", dict(rgba=True, rowbytes=4 * W, ostride=4 * W * H, tables=X, tstride=1008))]
    for what, kw in cases:
        assert call(**kw) == bb.E_INVALID, what
    assert fe.launch_count == launches and fe.last_kernel == kernel
    # a face layout without an origin for a plate of the globe the lensmap does not show (rectilinear at 60 degrees
    # shows one plate of the cube)
    fe.command("f_lens rectilinear")
    fe.command("f_fov 60")
    fe.build_lensmap(W, H, PS, threads=1)
    assert sum(fe.display()) == 1
    shown = fe.display().index(1)
    fe.set_face_layout(PS * (shown + 1), [(i * PS, 0) for i in range(shown + 1)])
    fe.warp_view(F, O, rowbytes=W, screen_stride=W * H, nframes=1, face_stride=PS * PS * 6)   # the lensmap's warp takes it
    torch.cuda.synchronize()
    launches = fe.launch_count
    assert call(fstride=PS * PS * 6) == bb.E_INVALID and "has no origin" in lib.blinky_last_error(fe._ctx).decode()
    fe.set_face_layout(6 * PS - 1, [(i * PS, 0) for i in range(6)])   # plate 5 does not fit
    assert call(fstride=PS * PS * 6) == bb.E_INVALID
    assert fe.launch_count == launches
    fe.set_face_layout()
    # a globe_plate globe, no globe, no lensmap: E_STATE
    fe.command("f_globe fast")
    assert call() == bb.E_STATE and "blinky_set_raymap_device" in lib.blinky_last_error(fe._ctx).decode()
    assert fe.launch_count == launches
    fresh = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        assert call(ctx=fresh._ctx) == bb.E_STATE
        fresh.command("f_globe cube")
        assert call(ctx=fresh._ctx) == bb.E_STATE, "no lensmap installed"
        assert fresh.launch_count == 0
    finally:
        fresh.close()


def test_plate_size_beyond_a_ray_map_is_refused(bb, torch, pair):
    """a supplied one-plate lensmap may have ps up to 16384, past what a ray map takes (6 * ps^2 < 2^28, ps <= 6688,
    which is also what the kernel's packed texel holds): refused with E_STATE, nothing launched; 6688 is taken"""
    fe, _ = pair
    fe.command("f_globe cube")
    w, h = 64, 32
    out = torch.zeros(w * h, dtype=torch.uint8, device="cuda")
    faces = torch.zeros(64, dtype=torch.uint8, device="cuda")   # (no ray below maps: nothing is read)
    rays = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
    rays[:, :, 2] = 1
    for ps in (8200, 6689):
        fe.set_lensmap(np.full((h, w), 0x70000000, np.uint32), ps, 1)
        launches = fe.launch_count
        with pytest.raises(bb.BlinkyError) as e:
            fe.warp_rays(faces, out, rays, face_stride=0)
        assert e.value.code == bb.E_STATE and "plate size" in str(e.value), str(e.value)
        assert fe.launch_count == launches
    fe.set_raymap(np.zeros((h, w, 3), np.float32), 6688)
    assert fe.platesize == 6688
    launches = fe.launch_count
    fe.warp_rays(faces, out, torch.zeros((h, w, 3), dtype=torch.float32, device="cuda"), face_stride=0)
    torch.cuda.synchronize()
    assert fe.launch_count == launches + 1


@pytest.mark.parametrize("form", ["8bit-rubix-quad", "rgba-keep-pixel", "one-matrix"])
def test_small_view_large_batch_splits_the_frames(bb, torch, pair, form):
    """A small view in a batch of 400 frames sharing one field: the frames are split over rows of threads so that the
    launch fills the GPU (96 x 64 quads: 2 frames per thread), each thread still reading its rays once"""
    fe, ref = pair
    rays = setup(pair, rubix=form.startswith("8bit"))
    n = 400
    distinct = matrices(5)
    which = np.arange(n) % len(distinct) if form != "one-matrix" else np.zeros(n, int)
    xs = distinct[which] if form != "one-matrix" else distinct[3]
    rgba = form.startswith("rgba")
    keep = "keep" in form
    quad = form != "rgba-keep-pixel"
    if rgba:
        table = np.random.default_rng(2).integers(0, 2**32, 256, dtype=np.uint32)
        for c in pair:
            c.set_rgba_table(table)
    scr = Screens(torch, n, rgba, x0=8 if quad else 3, y0=2, extra=12 if quad else 13)
    d_faces = faces_for(torch, fe, 1)
    out = scr.new()
    fe.warp_rays(d_faces, out.data_ptr(), torch.from_numpy(rays).cuda(), torch.from_numpy(np.ascontiguousarray(xs)).cuda(), x0=scr.x0, y0=scr.y0,
                 rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep, rgba=rgba, screen_stride=scr.stride, face_stride=0)
    torch.cuda.synchronize()
    kernel = fe.last_kernel
    fpt = int(kernel.split("frames/thread=")[1])
    assert 1 < fpt < n, kernel
    assert f"quad={int(quad)}" in kernel, kernel
    got = out.cpu().numpy()
    for f in sorted(set(range(0, n, 23)) | {1, 2, 3, n - 2, n - 1}):
        M = distinct[which[f]] if form != "one-matrix" else xs
        want = reference(torch, ref, rays, M, d_faces, scr, f, keep, rgba, None)
        bad = np.nonzero(got[f * scr.stride:(f + 1) * scr.stride] != want)[0]
        assert bad.size == 0, (kernel, f, bad.size)
    assert np.array_equal(got[n * scr.stride:], scr.fill.cpu().numpy()[n * scr.stride:])


# ---- 4K look-around ----------------------------------------------------------------------------------------------

def test_4k_look_around(bb, torch, pair):
    fe, ref = pair
    W4, H4, P4 = 3840, 2160, 2048
    for c in pair:
        c.command("f_globe cube")
        c.command("f_lens panini")
        c.command("f_fov 180")
        c.build_lensmap(W4, H4, P4, threads=0)
    d_rays = torch.empty((H4, W4, 3), dtype=torch.float32, device="cuda")
    fe.raymap(W4, H4, out=d_rays)
    torch.cuda.synchronize()
    n = 60
    xs = np.stack([yaw(6.0 * i) for i in range(n)])
    d_x = torch.from_numpy(xs).cuda()
    d_faces = torch.from_numpy(np.random.default_rng(0).integers(0, 256, 6 * P4 * P4, dtype=np.uint8)).cuda()
    out = torch.empty((n, H4, W4), dtype=torch.uint8, device="cuda")
    fe.warp_rays(d_faces, out, d_rays, d_x, face_stride=0)
    torch.cuda.synchronize()
    assert fe.last_kernel.startswith("ray_warp_kernel<quad=1,") and f"frames/thread={n}" in fe.last_kernel
    rays = d_rays.cpu().numpy()
    for f in (0, 17, 45, 59):
        ref.set_raymap(torch.from_numpy(turned(rays, xs[f])).cuda(), P4)
        want = torch.empty((H4, W4), dtype=torch.uint8, device="cuda")
        ref.warp(d_faces, want)
        torch.cuda.synchronize()
        assert torch.equal(out[f], want), f


# ---- adversarial rays, matrices and fields -----------------------------------------------------------------------

ARGMAX_GLOBES = ["cube", "cube_corner", "cube_edge", "tetra", "trism"]


def adversarial_matrices():
    """zero, singular, +-inf and NaN entries, 1e30 and subnormal 1e-40 entries, and exact 90-degree turns that take
    rays on plate edges and corners onto other plates' edges and corners"""
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    perm = np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]], np.float32)          # x -> y -> z -> x
    quarter = np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0]], np.float32)      # 90 degree yaw
    half_flip = np.array([[-1, 0, 0], [0, 0, -1], [0, -1, 0]], np.float32)  # reflection through a plate diagonal
    singular = np.array([[1, 2, 3], [2, 4, 6], [-1, 0.5, 0]], np.float32)
    with_inf = np.eye(3, dtype=np.float32)
    with_inf[0, 2] = inf
    with_inf[1, 1] = -inf
    with_nan = np.eye(3, dtype=np.float32)
    with_nan[2, 0] = nan
    huge = (np.eye(3) * 1e30).astype(np.float32)
    huge[0, 1] = -1e30
    tiny = np.full((3, 3), 1e-40, np.float32)
    tiny[2, 2] = 1
    return np.stack([np.zeros((3, 3), np.float32), singular, with_inf, with_nan, huge, tiny, perm, quarter, half_flip,
                     np.eye(3, dtype=np.float32)])


def adversarial_field(fe, ps, w, h):
    """test_raymap_host_only's adversarial rays (zeros, -0, NaN, +-inf, subnormals, +-3e38, u or v exactly 0 or 1, u * ps
    reaching ps, cube-corner ties) for the globe on `fe`, then the lens's own rays, as a [h, w, 3] field"""
    slots = np.zeros((6, 11), np.float32)
    pl = fe.plates()
    slots[: len(pl)] = pl
    rays = adversarial_rays(slots, len(pl), ps)
    extra = np.array([[-3e38, 3e38, 1], [-0.0, -0.0, 1], [1, -0.0, 0], [np.float32(1e-45), 1, 0], [1, 1, np.nan]], np.float32)
    rays = np.vstack([rays, extra])
    field = fe.raymap(w, h).reshape(-1, 3)
    assert len(rays) <= len(field), len(rays)
    field[: len(rays)] = rays
    return field.reshape(h, w, 3)


@pytest.mark.parametrize("quad", [True, False])
@pytest.mark.parametrize("globe", ARGMAX_GLOBES)
def test_adversarial_rays_and_matrices(bb, torch, pair, globe, quad):
    fe, ref = pair
    setup(pair, globe=globe, rubix=True, grid=(4, 3.0, 2.0))
    rays = adversarial_field(fe, PS, W, H)
    xs = adversarial_matrices()
    n = len(xs)
    d_faces = faces_for(torch, fe, n)
    scr = Screens(torch, n, False, x0=8 if quad else 3, y0=2, extra=12 if quad else 13)
    check_batch(torch, fe, ref, rays, xs, d_faces, scr, quad, False, expect_kernel=f"ray_warp_kernel<quad={int(quad)},rubix=1")
    # and not turned at all
    check_batch(torch, fe, ref, rays, None, d_faces, scr, not quad, False, expect_kernel=f"ray_warp_kernel<quad={int(quad)},rubix=1")


def warp_dense_against_the_rule(torch, fe, ref, rays, xs, w, h, ps, rgba=False):
    """warp_rays into dense [n, h, w] screens (quads where w allows) against set_raymap + warp_view, frame by frame"""
    n = len(xs)
    bpp = 4 if rgba else 1
    d_faces = torch.randint(0, 256, (n, fe.numplates * ps * ps), dtype=torch.uint8, device="cuda")
    out = torch.full((n * h * w * bpp,), 77, dtype=torch.uint8, device="cuda")
    fe.warp_rays(d_faces, out.data_ptr(), torch.from_numpy(rays).cuda(), torch.from_numpy(xs).cuda(), rowbytes=w * bpp,
                 screen_stride=w * h * bpp, nframes=n, rgba=rgba)
    torch.cuda.synchronize()
    kernel = fe.last_kernel
    got = out.cpu().numpy().reshape(n, -1)
    for f in range(n):
        with np.errstate(all="ignore"):
            ref.set_raymap(np.ascontiguousarray(turned(rays, xs[f])), ps)
        want = torch.full((h * w * bpp,), 77, dtype=torch.uint8, device="cuda")
        ref.warp_view(d_faces[f:f + 1], want.data_ptr(), rowbytes=w * bpp, screen_stride=w * h * bpp, nframes=1, rgba=rgba)
        torch.cuda.synchronize()
        bad = np.nonzero(got[f] != want.cpu().numpy())[0]
        assert bad.size == 0, (kernel, f, bad.size, bad[:8].tolist())
    return kernel


@pytest.mark.parametrize("lens,zoom,w,h", [("panini", "f_fov 360", 96, 64), ("mercator", "f_vfov 180", 96, 64),
                                           ("fisheye1", "f_contain", 8, 640), ("cylinder", "f_vfov 180", 1000, 8)])
def test_exported_fields_of_extreme_zooms(bb, torch, pair, lens, zoom, w, h):
    """the fields the exports give at the sweep's extreme zooms (panini at an infinite scale: lens_inverse of +-inf and
    NaN) turned by ordinary and adversarial matrices, rubix on with a non-default grid"""
    fe, ref = pair
    ps = 48
    for c in pair:
        c.set_rubixgrid(4, 3.0, 2.0)
        c.command("f_globe cube_corner")
        c.command(f"f_lens {lens}")
        c.command(zoom)
        c.set_rubix(True)
        c.build_lensmap(w, h, ps, threads=1)
        c.set_rgba_table(np.random.default_rng(2).integers(0, 2**32, 256, dtype=np.uint32))
    d = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
    fe.raymap(w, h, out=d)
    rays = d.cpu().numpy()
    xs = np.concatenate([matrices(4), adversarial_matrices()])
    for rgba in (False, True):
        kernel = warp_dense_against_the_rule(torch, fe, ref, rays, xs, w, h, ps, rgba=rgba)
        assert f"quad={int(w % 4 == 0)}" in kernel, kernel


def test_plate_size_at_the_texel_packing_limit(bb, torch, pair):
    """ps 6688, the largest plate a ray map takes: rays reaching u * ps = ps and the texels px, py = 6687 at every plate
    edge, in quads and per pixel"""
    fe, ref = pair
    ps = 6688
    for c in pair:
        c.set_rubixgrid(4, 3.0, 2.0)
        c.command("f_globe cube")
        c.set_rubix(True)
    slots = fe.plates()
    edge = u_one_rays(slots, len(slots), ps)
    # v = 1 too: the same rays with the plate's right and up exchanged
    flipped = []
    for plate in range(len(slots)):
        f, rt, up = (slots[plate][k:k + 3].astype(np.float64) for k in (0, 3, 6))
        t = np.tan(float(np.float32(slots[plate][9]) / np.float32(2)))
        for a in np.linspace(-0.9, 0.9, 5):
            base = f - up * t + rt * a * t
            flipped += [(base * (1 + k * 2.0 ** -24)).astype(np.float32) for k in range(-6, 7)]
    rays = np.vstack([edge, np.array(flipped, np.float32)])
    for w in (64, 62):
        h = -(-len(rays) // w)
        field = np.zeros((h * w, 3), np.float32)
        field[: len(rays)] = rays
        field[len(rays):] = [0, 0, 1]
        field = field.reshape(h, w, 3)
        for c in pair:
            c.set_raymap(field, ps)
        entries = fe.lensmap_packed().reshape(-1)
        texel = entries & 0x0FFFFFFF
        mapped = (entries >> 31) == 1
        px, py = texel % ps, texel // ps % ps
        assert (mapped & (px == ps - 1)).any() and (mapped & (py == ps - 1)).any()
        xs = np.stack([np.eye(3, dtype=np.float32), adversarial_matrices()[6], adversarial_matrices()[7]])
        kernel = warp_dense_against_the_rule(torch, fe, ref, field, xs, w, h, ps)
        assert f"quad={int(w % 4 == 0)}" in kernel, kernel
