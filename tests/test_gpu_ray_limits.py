"""The ray warps (blinky_warp_device_rays[_rgba], k = 1, and blinky_warp_device_rays_supersampled, k = 2, 3, 4) at the
limits of their index ranges and view shapes, against tests/ray_reference.py, which uses no project kernel.

Covered: views of 1 pixel, odd widths, partial last CTAs and rows or columns past 65536 pixels; adversarial rays and
matrices on every argmax globe through the supersampled warp; the exported k-fold fields of extreme zooms; plate size
6688; batches of 65535 frames and batches that frames_per_thread does not divide; output frames, output rows, face
frames, plate origins, fields, matrices and tables past 2^32 bytes, and per-frame fields, matrices and tables past
2^34; a field past 4 GiB; and the supersampled kernel's 31-bit field pixel index on both sides of its limit.

Every byte of each output buffer is compared: each checked frame's view against the reference, and everything else
(margins, unchecked views, the frames and bytes after the batch) against what the buffer held before the launch.  The
screens of the view-shape cases have 256 rows of margin below the view and frames after the batch, so that a broken
bounds guard shows up as changed margin bytes inside the allocation.  The cases past 4 GiB allocate up to about 9 GB,
the 31-bit case about 25 GB (skipped, alone, when the device has less free memory)."""
import gc

import numpy as np
import pytest

import ray_reference as rr
from test_gpu_ray_warp import adversarial_matrices, matrices, yaw
from test_raymap_host_only import adversarial_rays, u_one_rays

pytestmark = pytest.mark.gpu

PS = 48
GRID = (4, 3.0, 2.0)
TABLE = np.random.default_rng(2).integers(0, 2**32, 256, dtype=np.uint32)
SENTINEL = 0x5A
ARGMAX_GLOBES = ["cube", "cube_corner", "cube_edge", "tetra", "trism"]


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture(autouse=True)
def _free_device_memory(torch):
    yield
    gc.collect()
    torch.cuda.empty_cache()


class Case:
    """a device context with an all-unmapped w x h map of plate size ps installed (the ray warps read only its size,
    plate size and background), and a host-only context on the same globe, rubix state and grid"""

    def __init__(self, torch, bb, palette, w, h, ps=PS, globe="cube", rubix=False, grid=None, seed=3):
        self.torch = torch
        self.fe = bb.Fisheye(device=0, palette=palette)
        if grid:
            self.fe.set_rubixgrid(*grid)
        self.fe.command(f"f_globe {globe}")
        self.fe.set_rubix(rubix)
        self.fe.set_rgba_table(TABLE)
        self.g = rr.HostGlobe(bb, palette, globe, rubix, grid)
        self.ps = ps
        self.install(w, h, seed)

    def install(self, w, h, seed=3):
        self.w, self.h = w, h
        self.fe.set_lensmap(np.full((h, w), 0x70000000, np.uint32), self.ps, self.fe.numplates)
        self.bg = np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)
        self.fe.set_background(self.bg.reshape(-1))

    def close(self):
        self.fe.close()
        self.g.close()

    def distinct(self, seed=0):
        """PERIOD distinct rays: the globe's adversarial rays and the panini rays of a small view"""
        slots = np.zeros((6, 11), np.float32)
        pl = self.g.fe.plates()
        slots[: len(pl)] = pl
        adv = adversarial_rays(slots, len(pl), self.ps)
        self.g.fe.command("f_lens panini")
        self.g.fe.command("f_fov 180")
        lens = self.g.fe.raymap(48, 32).reshape(-1, 3)
        rays = np.vstack([adv[::2], lens])
        rng = np.random.default_rng(seed)
        return np.ascontiguousarray(rays[rng.permutation(len(rays))[: rr.PERIOD]])

    def warp(self, k, rgba, d_faces, scr, d_rays, d_x, n, keep=False, tables=None, face_stride=None):
        """one launch into scr; its last_kernel"""
        launches = self.fe.launch_count
        self.fe.warp_rays(d_faces, scr.buf.data_ptr(), d_rays, d_x, x0=scr.x0, y0=scr.y0, rowbytes=scr.rowbytes, nframes=n, keep_unmapped=keep,
                          rgba=rgba, tables=tables, screen_stride=scr.stride, supersample=k, face_stride=face_stride)
        self.torch.cuda.synchronize()
        assert self.fe.launch_count == launches + 1
        return self.fe.last_kernel


@pytest.fixture()
def cases(bb, palette, torch):
    made = []

    def make(*a, **kw):
        made.append(Case(torch, bb, palette, *a, **kw))
        return made[-1]

    yield make
    for c in made:
        c.close()


class Screens:
    """n frames of screens of `stride` bytes, rows of `rowbytes`, a w x h view at (x0, y0); random bytes, or a
    constant byte for buffers of gigabytes.  `total`: the bytes allocated (default: n + frames_after frames)."""

    def __init__(self, torch, w, h, bpp, n, x0=0, y0=0, extra=0, rows_after=rr.MARGIN_ROWS, frames_after=None, rowbytes=None, stride=None,
                 total=None, const=None, seed=9):
        self.torch, self.w, self.h, self.bpp, self.n, self.x0, self.y0 = torch, w, h, bpp, n, x0, y0
        self.rowbytes = rowbytes or (x0 + w + extra) * bpp
        self.stride = stride or (y0 + h + rows_after) * self.rowbytes
        total = total or (n + (n if frames_after is None else frames_after)) * self.stride
        assert total >= (n - 1) * self.stride + (y0 + h - 1) * self.rowbytes + (x0 + w) * bpp
        self.const = const
        if const is None:
            g = torch.Generator(device="cuda")
            g.manual_seed(seed)
            self.fill = torch.randint(0, 256, (total,), dtype=torch.uint8, device="cuda", generator=g)
            self.buf = self.fill.clone()
        else:
            self.fill = None
            self.buf = torch.full((total,), const, dtype=torch.uint8, device="cuda")

    def views(self, t):
        return t.as_strided((self.n, self.h, self.w * self.bpp), (self.stride, self.rowbytes, 1), self.y0 * self.rowbytes + self.x0 * self.bpp)

    def check(self, refs, what):
        """refs: {frame: (pixels, written)} by the reference; then every other byte of the buffer as it was"""
        got = self.views(self.buf)
        for f, (pix, written) in refs.items():
            have = got[f].cpu().numpy().reshape(self.h, self.w, self.bpp)
            if self.fill is None:
                base = np.full_like(have, self.const)
            else:
                base = self.views(self.fill)[f].cpu().numpy().reshape(have.shape)
            want = np.where(written[..., None], pix.reshape(have.shape), base)
            bad = np.argwhere((have != want).any(-1))
            assert bad.size == 0, (what, f, len(bad), bad[:8].tolist())
        # the views restored to what they held, every byte of the buffer
        if self.fill is None:
            got.fill_(self.const)
            step = 1 << 28
            for i in range(0, self.buf.numel(), step):
                assert bool((self.buf[i:i + step] == self.const).all()), (what, "bytes outside the views changed near", i)
        else:
            got.copy_(self.views(self.fill))
            diff = (self.buf != self.fill).nonzero().flatten()
            assert diff.numel() == 0, (what, "bytes outside the views changed", diff.numel(), diff[:8].tolist())


def fpt_of(kernel):
    return int(kernel.split("frames/thread=")[1])


def expect_instance(kernel, k, rgba, quad=None, rubix=None, keep=None, tables=None):
    if k > 1:
        assert kernel.startswith(f"ray_supersample_kernel<k={k},"), kernel
    else:
        assert kernel.startswith("ray_warp_kernel<") and f"rgba={int(rgba)}" in kernel, kernel
        if quad is not None:
            assert f"quad={int(quad)}" in kernel, kernel
    for name, v in (("rubix", rubix), ("keep", keep), ("tables", tables)):
        if v is not None:
            assert f"{name}={int(v)}," in kernel or f"{name}={int(v)}>" in kernel, kernel


def dense_faces(torch, fe, n, ps, seed=1):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randint(0, 256, (n, fe.numplates * ps * ps), dtype=torch.uint8, device="cuda", generator=g)


# ---- view shapes -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("shape", rr.SHAPES, ids=[f"{w}x{h}" for w, h in rr.SHAPES])
def test_view_shapes(bb, torch, cases, shape, k):
    """every view shape through every factor, keep_unmapped off and on: the last partial CTA and the pix >= nitems
    guard (every shape but 8 x 640 has a partial last CTA), 1-pixel rows and columns, rows and columns past 65536"""
    w, h = shape
    i = rr.SHAPES.index(shape)
    rubix = (i + k) % 2 == 1
    rgba = k > 1 or i % 2 == 1
    bpp = 4 if rgba else 1
    x0 = 3 if (i + k) % 3 == 0 else 4
    c = cases(w, h, rubix=rubix, grid=GRID if rubix else None, seed=i)
    n = 2
    D = c.distinct(seed=i)
    field = D[np.arange(k * k * w * h) % rr.PERIOD].reshape(k * h, k * w, 3)
    # every 7th pixel wholly unmapped (its samples zero rays)
    blocks = field.reshape(h, k, w, k, 3).transpose(0, 2, 1, 3, 4)
    blocks[(np.arange(w * h) % 7 == 3).reshape(h, w)] = 0
    xs = matrices(n, seed=i)
    d_rays, d_x = torch.from_numpy(field).cuda(), torch.from_numpy(xs).cuda()
    d_faces = dense_faces(torch, c.fe, n, PS, seed=i)
    faces = d_faces.cpu().numpy()
    extra = (-(x0 + w)) % 4 + 4
    refs = {f: rr.frame(c.g, field, xs[f], faces[f], c.bg, k, PS, table=TABLE if rgba else None) for f in range(n)}
    for keep in (False, True):
        scr = Screens(torch, w, h, bpp, n, x0=x0, y0=1, extra=extra, seed=i + 17 * keep)
        kernel = c.warp(k, rgba, d_faces, scr, d_rays, d_x, n, keep=keep)
        expect_instance(kernel, k, rgba, quad=w % 4 == 0 and x0 % 4 == 0, rubix=rubix, keep=keep)
        scr.check({f: (p, wr if keep else np.ones_like(wr)) for f, (p, wr) in refs.items()}, (kernel, keep))
    if k > 1 and w * h > 1:
        assert any(wr.any() and not wr.all() for _, wr in refs.values()), "some pixels wholly unmapped, some not"


# ---- adversarial rays and matrices, supersampled -----------------------------------------------------------------

@pytest.mark.parametrize("k", [2, 4])
@pytest.mark.parametrize("globe", ARGMAX_GLOBES)
def test_adversarial_rays_and_matrices(bb, torch, cases, globe, k):
    """the adversarial rays spread over sub-samples (every third sample), so that pixels mix them with the lens's
    rays, turned by the adversarial matrices"""
    w, h = 96, 64
    c = cases(w, h, globe=globe, rubix=True, grid=GRID)
    slots = np.zeros((6, 11), np.float32)
    pl = c.g.fe.plates()
    slots[: len(pl)] = pl
    adv = np.vstack([adversarial_rays(slots, len(pl), PS),
                     np.array([[-3e38, 3e38, 1], [-0.0, -0.0, 1], [1, -0.0, 0], [np.float32(1e-45), 1, 0], [1, 1, np.nan]], np.float32)])
    c.g.fe.command("f_lens panini")
    c.g.fe.command("f_fov 180")
    field = c.g.fe.raymap(k * w, k * h)
    flat = field.reshape(-1, 3)
    at = np.arange(len(adv)) * 3 + 1
    assert at[-1] < len(flat)
    flat[at] = adv
    xs = adversarial_matrices()
    n = len(xs)
    keep = k == 4
    d_faces = dense_faces(torch, c.fe, n, PS)
    faces = d_faces.cpu().numpy()
    scr = Screens(torch, w, h, 4, n, x0=5, y0=2, extra=3, rows_after=2)
    kernel = c.warp(k, True, d_faces, scr, torch.from_numpy(field).cuda(), torch.from_numpy(xs).cuda(), n, keep=keep)
    expect_instance(kernel, k, True, rubix=True, keep=keep, tables=False)
    refs = {}
    for f in range(n):
        pix, wr = rr.frame(c.g, field, xs[f], faces[f], c.bg, k, PS, table=TABLE)
        refs[f] = (pix, wr if keep else np.ones_like(wr))
    scr.check(refs, kernel)


# ---- exported k-fold fields of extreme zooms ---------------------------------------------------------------------

@pytest.mark.parametrize("k", [2, 4])
@pytest.mark.parametrize("lens,zoom,w,h", [("panini", "f_fov 360", 96, 64), ("mercator", "f_vfov 180", 96, 64),
                                           ("fisheye1", "f_contain", 8, 640), ("cylinder", "f_vfov 180", 1000, 8)])
def test_exported_fields_of_extreme_zooms(bb, torch, cases, lens, zoom, w, h, k):
    """fe.raymap(k w, k h) at the zoom sweep's extremes (panini at an infinite scale: NaN and infinite rays) on the
    cube_corner globe, turned by ordinary and adversarial matrices"""
    c = cases(w, h, globe="cube_corner", rubix=True, grid=GRID)
    c.fe.command(f"f_lens {lens}")
    c.fe.command(zoom)
    d_rays = torch.empty((k * h, k * w, 3), dtype=torch.float32, device="cuda")
    c.fe.raymap(k * w, k * h, out=d_rays)
    torch.cuda.synchronize()
    field = d_rays.cpu().numpy()
    xs = np.concatenate([matrices(4), adversarial_matrices()])
    n = len(xs)
    d_faces = dense_faces(torch, c.fe, n, PS)
    faces = d_faces.cpu().numpy()
    scr = Screens(torch, w, h, 4, n, x0=1, y0=1, extra=2, rows_after=2)
    kernel = c.warp(k, True, d_faces, scr, d_rays, torch.from_numpy(xs).cuda(), n)
    expect_instance(kernel, k, True, rubix=True, keep=False)
    refs = {}
    for f in range(n):
        pix, wr = rr.frame(c.g, field, xs[f], faces[f], c.bg, k, PS, table=TABLE)
        refs[f] = (pix, np.ones_like(wr))
    scr.check(refs, kernel)


# ---- plate size 6688 ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [2, 4])
def test_plate_size_at_the_texel_packing_limit(bb, torch, cases, k):
    """ps 6688 through the supersampled warp: rays a few ulps either side of u = 1 and of v = 1 on every plate, so that
    samples land on px or py = 6687 at every plate edge"""
    ps = 6688
    c = cases(16, 8, ps=ps, rubix=True, grid=GRID)
    slots = c.g.fe.plates()
    edge = u_one_rays(slots, len(slots), ps)
    flipped = []
    for plate in range(len(slots)):
        f, rt, up = (slots[plate][j:j + 3].astype(np.float64) for j in (0, 3, 6))
        t = np.tan(float(np.float32(slots[plate][9]) / np.float32(2)))
        for a in np.linspace(-0.9, 0.9, 5):
            base = f - up * t + rt * a * t
            flipped += [(base * (1 + j * 2.0 ** -24)).astype(np.float32) for j in range(-6, 7)]
    rays = np.vstack([edge, np.array(flipped, np.float32)])
    w = 16
    fw = k * w
    h = -(-len(rays) // (fw * k))
    c.install(w, h)
    field = np.zeros((k * h * fw, 3), np.float32)
    field[: len(rays)] = rays
    field[len(rays):] = [0, 0, 1]
    field = field.reshape(k * h, fw, 3)
    xs = np.stack([np.eye(3, dtype=np.float32), adversarial_matrices()[6], adversarial_matrices()[7]])
    n = len(xs)
    rng = np.random.default_rng(4)
    faces = rng.integers(0, 256, 6 * ps * ps, dtype=np.uint8)
    d_faces = torch.from_numpy(faces).cuda()
    scr = Screens(torch, w, h, 4, n, x0=3, y0=1, extra=1, rows_after=2)
    kernel = c.warp(k, True, d_faces, scr, torch.from_numpy(field).cuda(), torch.from_numpy(xs).cuda(), n, keep=True, face_stride=0)
    expect_instance(kernel, k, True, rubix=True, keep=True)
    refs = {}
    edges = [0, 0]
    for f in range(n):
        idx, tint = c.g.texels(field, ps, xs[f])
        m = idx >= 0
        edges[0] += int((m & (idx % ps == ps - 1)).sum())
        edges[1] += int((m & (idx // ps % ps == ps - 1)).sum())
        refs[f] = rr.colour(c.g, idx, tint, faces, c.bg, k, ps, table=TABLE)
    assert edges[0] and edges[1], edges
    scr.check(refs, kernel)


# ---- batches -----------------------------------------------------------------------------------------------------

def checked_frames(n):
    return sorted({0, 1, n - 2, n - 1} | set(range(0, n, 97)))


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("form", ["matrices", "fields"])
def test_65535_frames(bb, torch, cases, form, k):
    """the most frames a launch takes, of a 3 x 2 view, with per-frame matrices (one field) or per-frame fields (no
    turn): one frame per row of threads, grid.y = 65535"""
    w, h, n = 3, 2, rr.MAX_FRAMES
    c = cases(w, h, rubix=True)
    D = c.distinct()
    nf = k * k * w * h
    if form == "matrices":
        a = np.radians(np.arange(n) * 0.61)
        xs = np.zeros((n, 3, 3), np.float32)
        xs[:, 0, 0], xs[:, 0, 2], xs[:, 1, 1], xs[:, 2, 0], xs[:, 2, 2] = np.cos(a), np.sin(a), 1, -np.sin(a), np.cos(a)
        field = D[np.arange(nf) % rr.PERIOD].reshape(k * h, k * w, 3)
        d_rays, d_x = torch.from_numpy(field).cuda(), torch.from_numpy(xs).cuda()
    else:
        d_rays = torch.empty((n, k * h, k * w, 3), dtype=torch.float32, device="cuda")
        rr.fill_tiled(torch, d_rays, D)
        d_x = None
    d_faces = dense_faces(torch, c.fe, 1, PS)
    faces = d_faces.cpu().numpy()[0]
    scr = Screens(torch, w, h, 4, n, x0=1, y0=1, extra=2, rows_after=2, frames_after=4)
    kernel = c.warp(k, True, d_faces, scr, d_rays, d_x, n, face_stride=0)
    expect_instance(kernel, k, True, quad=False, rubix=True, keep=False)
    assert fpt_of(kernel) == 1 and f"grid=(1,{n})" in kernel, kernel
    refs = {}
    base_idx, base_tint = c.g.texels(D, PS)
    for f in checked_frames(n):
        if form == "matrices":
            pix, wr = rr.frame(c.g, field, xs[f], faces, c.bg, k, PS, table=TABLE)
        else:
            idx, tint = rr.tiled_texels(base_idx, base_tint, 0, k * h, k * w, offset=f * nf)
            pix, wr = rr.colour(c.g, idx, tint, faces, c.bg, k, PS, table=TABLE)
        refs[f] = (pix, np.ones_like(wr))
    scr.check(refs, kernel)


@pytest.mark.parametrize("k", [1, 3])
def test_batch_that_frames_per_thread_does_not_divide(bb, torch, cases, k):
    """997 frames sharing one field, turned by a cycle of matrices: the last row of threads carries fewer frames"""
    w, h, n = 96, 64, rr.ODD_BATCH
    c = cases(w, h, rubix=False)
    D = c.distinct(seed=5)
    field = D[np.arange(k * k * w * h) % rr.PERIOD].reshape(k * h, k * w, 3)
    distinct = matrices(5)
    xs = np.ascontiguousarray(distinct[np.arange(n) % 5])
    d_faces = dense_faces(torch, c.fe, 1, PS)
    faces = d_faces.cpu().numpy()[0]
    scr = Screens(torch, w, h, 4, n, x0=1, y0=2, extra=3, rows_after=2, frames_after=64)
    kernel = c.warp(k, True, d_faces, scr, torch.from_numpy(field).cuda(), torch.from_numpy(xs).cuda(), n, keep=True, face_stride=0)
    fpt = fpt_of(kernel)
    assert 1 < fpt <= 64 and n % fpt != 0, kernel
    assert f",{-(-n // fpt)}) block" in kernel, kernel
    expect_instance(kernel, k, True, quad=False, keep=True)
    per = {m: rr.frame(c.g, field, distinct[m], faces, c.bg, k, PS, table=TABLE) for m in range(5)}
    scr.check({f: per[f % 5] for f in checked_frames(n)}, kernel)


@pytest.mark.parametrize("k", [1, 2])
def test_65536_frames_are_refused(bb, torch, cases, k):
    w, h = 3, 2
    c = cases(w, h)
    d_rays = torch.zeros((k * h, k * w, 3), dtype=torch.float32, device="cuda")
    d_x = torch.eye(3, dtype=torch.float32, device="cuda").expand(rr.MAX_FRAMES + 1, 3, 3).contiguous()
    out = torch.zeros(16, dtype=torch.uint8, device="cuda")
    launches, kernel = c.fe.launch_count, c.fe.last_kernel
    with pytest.raises(bb.BlinkyError) as e:
        c.fe.warp_rays(torch.zeros(64, dtype=torch.uint8, device="cuda"), out, d_rays, d_x, rgba=True, rowbytes=4 * w, screen_stride=0,
                       supersample=k, face_stride=0)
    assert e.value.code == bb.E_INVALID and "65535" in str(e.value), str(e.value)
    assert c.fe.launch_count == launches and c.fe.last_kernel == kernel
    assert int(out.sum()) == 0


# ---- past 4 GiB --------------------------------------------------------------------------------------------------

LIMITS = ["frame", "pitch", "faces", "plate", "rays", "xforms", "tables"]


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("limit", LIMITS)
def test_past_4_gib(bb, torch, cases, limit, k):
    """one offset past 2^32 bytes at a time (k = 1: RGBA).  The fields tile PERIOD distinct rays, and the gaps of each
    strided allocation hold something else, so that a wrapped offset reads or writes other bytes."""
    w, h = rr.LIMIT_VIEW
    if limit == "pitch":
        h = rr.PITCH_ROWS
    c = cases(w, h, rubix=True, grid=GRID)
    D = c.distinct(seed=2)
    base_idx, base_tint = c.g.texels(D, PS)
    kh, kw = k * h, k * w
    n, face_stride, tables, layout = 1, 0, None, None
    offsets = [0]                 # per frame: the tiling offset of its field
    M = [yaw(0)]                  # per frame: its matrix
    d_faces = dense_faces(torch, c.fe, 1, PS)
    frame_faces = [d_faces[0].cpu().numpy()]
    d_rays = torch.empty((kh, kw, 3), dtype=torch.float32, device="cuda")
    rr.fill_tiled(torch, d_rays, D)
    d_x = torch.from_numpy(M[0]).cuda()
    scr_kw = dict(rows_after=2, frames_after=1, const=SENTINEL)
    if limit == "frame":
        n = rr.OUT_FRAMES
        stride = rr.OUT_STRIDE
        assert (n - 1) * stride > rr.GiB4
        scr = Screens(torch, w, h, 4, n, x0=1, y0=1, stride=stride, rowbytes=4 * (w + 4),
                      total=(n - 1) * stride + (h + 3) * 4 * (w + 4), const=SENTINEL)
        offsets, M, frame_faces = offsets * n, M * n, frame_faces * n
    elif limit == "pitch":
        scr = Screens(torch, w, h, 4, 1, x0=0, y0=0, rowbytes=rr.MAX_PITCH, stride=h * rr.MAX_PITCH, total=(h - 1) * rr.MAX_PITCH + 4 * w + 4096,
                      const=SENTINEL)
        assert (h - 1) * rr.MAX_PITCH >= rr.GiB4
    else:
        scr = Screens(torch, w, h, 4, 2 if limit != "plate" else 1, x0=2, y0=1, extra=1, **scr_kw)
    if limit == "faces":
        n, face_stride = 2, rr.FACE_STRIDE
        fb = 6 * PS * PS
        d_faces = torch.randint(0, 256, (face_stride + fb,), dtype=torch.uint8, device="cuda")
        frame_faces = [d_faces[f * face_stride:f * face_stride + fb].cpu().numpy() for f in range(n)]
        offsets, M = offsets * n, M * n
    elif limit == "plate":
        rb = rr.PLATE_ROWBYTES
        origins = [(i * PS, 0) for i in range(5)] + [(rr.PLATE_X, rr.PLATE_Y)]
        layout = (rb, origins)
        c.fe.set_face_layout(rb, origins)
        d_faces = torch.randint(0, 256, ((rr.PLATE_Y + PS) * rb,), dtype=torch.uint8, device="cuda")
        frame_faces = [d_faces]
        face_stride = d_faces.numel()
        assert rr.PLATE_Y * rb + rr.PLATE_X > rr.GiB4
        assert ((base_idx >= 0) & (base_idx // (PS * PS) == 5)).any(), "no ray on plate 5"
    elif limit == "rays":
        n = 2
        fb = rr.field_bytes(k, w, h)
        store = torch.empty(((rr.RAY_STRIDE + fb) // 4,), dtype=torch.float32, device="cuda")
        rr.fill_tiled(torch, store.view(-1)[: store.numel() // 3 * 3].view(-1, 3), D, offset=500)
        d_rays = store.as_strided((n, kh, kw, 3), (rr.RAY_STRIDE // 4, 3 * kw, 3, 1))
        offsets = [0, 7]
        for f in range(n):
            rr.fill_tiled(torch, d_rays[f], D, offset=offsets[f])
        M = M * n
        d_x = torch.from_numpy(M[0]).cuda()
    elif limit == "xforms":
        n = 2
        store = torch.full(((rr.XFORM_STRIDE + 36) // 4,), 0.25, dtype=torch.float32, device="cuda")
        M = [yaw(30), matrices(3)[1]]
        d_x = store.as_strided((n, 3, 3), (rr.XFORM_STRIDE // 4, 3, 1))
        d_x.copy_(torch.from_numpy(np.stack(M)))
        offsets = offsets * n
    elif limit == "tables":
        n = 2
        store = torch.randint(-2**31, 2**31 - 1, ((rr.TABLE_STRIDE + 1024) // 4,), dtype=torch.int32, device="cuda")
        tables = store.as_strided((n, 256), (rr.TABLE_STRIDE // 4, 1))
        offsets, M = offsets * n, M * n
    if limit in ("faces", "rays", "xforms", "tables"):
        frame_faces = frame_faces if limit == "faces" else frame_faces * n
    kernel = c.warp(k, True, d_faces, scr, d_rays, d_x, n, tables=tables, face_stride=face_stride)
    expect_instance(kernel, k, True, rubix=True, keep=False, tables=limit == "tables")
    refs = {}
    for f in range(n):
        t_idx, t_tint = c.g.texels(D, PS, M[f])
        idx, tint = rr.tiled_texels(t_idx, t_tint, 0, kh, kw, offset=offsets[f])
        table = TABLE if tables is None else tables[f].cpu().numpy().view(np.uint32)
        pix, wr = rr.colour(c.g, idx, tint, frame_faces[f], c.bg, k, PS, layout=layout, table=table)
        refs[f] = (pix, np.ones_like(wr))
    scr.check(refs, kernel)


def test_field_past_4_gib(bb, torch, cases):
    """k = 4 on a 6144 x 3648 view: one field of 4.3 GB; the first, a middle and the last 64 rows (the last hold the
    rays past 2^32 bytes) against the reference, every other byte of the screen as it was"""
    k = 4
    w, h = rr.BIG_VIEW
    ps = 256
    c = cases(w, h, ps=ps, rubix=True, grid=GRID)
    D = c.distinct(seed=6)
    base_idx, base_tint = c.g.texels(D, ps)
    d_rays = torch.empty((k * h, k * w, 3), dtype=torch.float32, device="cuda")
    rr.fill_tiled(torch, d_rays, D)
    rng = np.random.default_rng(8)
    faces = rng.integers(0, 256, 6 * ps * ps, dtype=np.uint8)
    scr = Screens(torch, w, h, 4, 1, rows_after=1, frames_after=0, const=SENTINEL)
    kernel = c.warp(k, True, torch.from_numpy(faces).cuda(), scr, d_rays, None, 1, face_stride=0)
    expect_instance(kernel, k, True, rubix=True, keep=False)
    del d_rays
    got = scr.views(scr.buf)[0]
    for y0 in (0, h // 2, h - 64):
        idx, tint = rr.tiled_texels(base_idx, base_tint, k * y0, k * 64, k * w)
        bg = np.ascontiguousarray(c.bg[y0:y0 + 64])
        pix, _ = rr.colour(c.g, idx, tint, faces, bg, k, ps, table=TABLE)
        have = got[y0:y0 + 64].cpu().numpy().reshape(64, w, 4)
        bad = np.argwhere((have != pix).any(-1))
        assert bad.size == 0, (kernel, y0, len(bad), bad[:8].tolist())
    got.fill_(SENTINEL)
    assert bool((scr.buf == SENTINEL).all())


# ---- the supersampled kernel's 31-bit field pixel index ----------------------------------------------------------

def test_31_bit_field_index(bb, torch, cases):
    """k = 4: 16384 x 8192 (k^2 W H = 2^31) is refused with E_INVALID and nothing launched; 16384 x 8191 (2^31 - 2^18)
    runs, its first, middle and last 8 rows against the reference.  The same 24 GiB then holds per-frame fields,
    matrices and tables 2^33 bytes apart, so that frame 2 starts past 2^34 bytes, for k = 1 and k = 4."""
    k = rr.FIELD_LIMIT_K
    W, H = rr.REFUSED_VIEW
    field_elems = 3 * k * k * W * H
    need = 4 * field_elems + 4 * W * H + (1 << 30)
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"the 31-bit field case needs {need} bytes of free device memory; the device reports {free} free of {total}")
    c = cases(W, H, rubix=True, grid=GRID)
    D = c.distinct(seed=9)
    base_idx, base_tint = c.g.texels(D, PS)
    store = torch.empty((field_elems,), dtype=torch.float32, device="cuda")
    out = torch.full((4 * W * H + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    faces = np.random.default_rng(3).integers(0, 256, 6 * PS * PS, dtype=np.uint8)
    d_faces = torch.from_numpy(faces).cuda()
    # refused: every buffer sized for the call
    rays = store.view(k * H, k * W, 3)
    launches, last = c.fe.launch_count, c.fe.last_kernel
    with pytest.raises(bb.BlinkyError) as e:
        c.fe.warp_rays(d_faces, out, rays, None, rowbytes=4 * W, screen_stride=0, rgba=True, supersample=k, face_stride=0)
    assert e.value.code == bb.E_INVALID and "31-bit" in str(e.value) and str(2**31) in str(e.value), str(e.value)
    assert c.fe.launch_count == launches and c.fe.last_kernel == last
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())
    # taken: one row less
    W, H = rr.TAKEN_VIEW
    c.install(W, H)
    rays = store[: 3 * k * k * W * H].view(k * H, k * W, 3)
    rr.fill_tiled(torch, rays, D)
    launches = c.fe.launch_count
    c.fe.warp_rays(d_faces, out, rays, None, rowbytes=4 * W, screen_stride=0, rgba=True, supersample=k, face_stride=0)
    torch.cuda.synchronize()
    assert c.fe.launch_count == launches + 1
    kernel = c.fe.last_kernel
    expect_instance(kernel, k, True, rubix=True, keep=False)
    got = out[: 4 * W * H].view(H, W, 4)
    for y0 in (0, H // 2, H - 8):
        idx, tint = rr.tiled_texels(base_idx, base_tint, k * y0, k * 8, k * W)
        pix, _ = rr.colour(c.g, idx, tint, faces, np.ascontiguousarray(c.bg[y0:y0 + 8]), k, PS, table=TABLE)
        have = got[y0:y0 + 8].cpu().numpy()
        bad = np.argwhere((have != pix).any(-1))
        assert bad.size == 0, (kernel, y0, len(bad), bad[:8].tolist())
    assert bool((out[4 * W * H:] == SENTINEL).all())
    del got, out, rays
    # per-frame fields, matrices and tables FAR_STRIDE apart, frame 2 past 2^34 bytes, in the same memory
    w, h = rr.LIMIT_VIEW
    c.install(w, h)
    S, n = rr.FAR_STRIDE // 4, rr.FAR_FRAMES
    assert (n - 1) * S + 3 * 16 * w * h + 1024 <= store.numel()
    rr.fill_tiled(torch, store[: store.numel() // 3 * 3].view(-1, 3), D, offset=300)
    M = [yaw(20), matrices(3)[1], yaw(-75)]
    for kk in (1, 4):
        d_rays = store.as_strided((n, kk * h, kk * w, 3), (S, 3 * kk * w, 3, 1))
        for f in range(n):
            rr.fill_tiled(torch, d_rays[f], D, offset=11 * f)
        # each frame's matrix and table just after its field
        d_x = store.as_strided((n, 3, 3), (S, 3, 1), 3 * kk * kk * w * h + 64)
        d_x.copy_(torch.from_numpy(np.stack(M)))
        tables = store.view(torch.int32).as_strided((n, 256), (S, 1), 3 * kk * kk * w * h + 128)
        tabs = np.random.default_rng(kk).integers(0, 2**32, (n, 256), dtype=np.uint32)
        tables.copy_(torch.from_numpy(tabs.view(np.int32)))
        scr = Screens(torch, w, h, 4, n, x0=1, y0=1, extra=3, rows_after=2)
        kernel = c.warp(kk, True, d_faces, scr, d_rays, d_x, n, tables=tables, face_stride=0)
        expect_instance(kernel, kk, True, rubix=True, keep=False, tables=True)
        refs = {}
        for f in range(n):
            t_idx, t_tint = c.g.texels(D, PS, M[f])
            idx, tint = rr.tiled_texels(t_idx, t_tint, 0, kk * h, kk * w, offset=11 * f)
            pix, wr = rr.colour(c.g, idx, tint, faces, c.bg, kk, PS, table=tabs[f])
            refs[f] = (pix, np.ones_like(wr))
        scr.check(refs, (kernel, "strides past 2^34"))
