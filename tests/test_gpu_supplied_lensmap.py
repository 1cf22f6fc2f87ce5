"""Supplied lensmaps on the GPU: blinky_set_lensmap_device plans a map that is already in device memory.

Its tile plan must be the host planner's byte for byte (the plan blinky_set_lensmap of the same map makes), and
every warp through it must write exactly what the same map supplied from host memory writes: the ring kernel, K3,
K1 and K0, 8-bit and RGBA, per-frame tables, keep_unmapped, views, a 3x2 atlas face layout, 1 / 5 / 16 frames and
warp_host.  The map is read in stream order, a refused map leaves the old one warping, and a graph captured before
the call keeps rendering the map it captured."""
import numpy as np
import pytest

from conftest import ALL_LENSES
from test_supplied_lensmap_host_only import RANDOM_KINDS, TINT_NONE, VALID, random_map, refusals

pytestmark = pytest.mark.gpu

KERNEL = {"ring": "warp_ring_kernel", "K1": "warp_gather_kernel", "K0": "warp_scalar_kernel", "K3": "warp_tile_gather_kernel"}
ZOOM = {"panini": "f_fov 180", "stereographic": "f_fov 180", "equirect": "f_contain", "hammer": "f_contain", "fisheye1": "f_contain",
        "quincuncial": "f_cover"}
BASELINE_4K = [("cube", "panini", False), ("cube", "stereographic", False), ("cube", "equirect", False), ("cube", "hammer", False),
               ("cube", "fisheye1", False), ("cube", "quincuncial", True), ("trism", "stereographic", False)]


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture()
def pair(bb, palette, cuda_device, monkeypatch):
    """(a context fed from host memory, one fed from device memory, one fed from device memory that launches
    GATHER tiles in their own kernel K3)"""
    a = bb.Fisheye(device=cuda_device, palette=palette)
    b = bb.Fisheye(device=cuda_device, palette=palette)
    monkeypatch.setenv("BLINKY_SERIAL_GATHER", "1")
    b3 = bb.Fisheye(device=cuda_device, palette=palette)
    monkeypatch.delenv("BLINKY_SERIAL_GATHER")
    yield a, b, b3
    for f in (a, b, b3):
        f.close()


def built_map(bb, palette, globe, lens, zoom, size, rubix=False, threads=8, device=None):
    fe = bb.Fisheye(device=device, palette=palette)
    try:
        fe.command(f"f_globe {globe}")
        fe.command(f"f_lens {lens}")
        if zoom:
            fe.command(zoom)
        fe.set_rubix(rubix)
        fe.build_lensmap(*size, threads=threads)
        return fe.lensmap_packed(), fe.numplates
    finally:
        fe.close()


def plan_of(fe):
    tiles, entries = fe.tile_plan()
    return tiles.tobytes(), entries.tobytes()


def assert_same_plan(torch, a, b, m, ps, n):
    a.set_lensmap(m, ps, n)
    b.set_lensmap(torch.from_numpy(m.view(np.int32)).cuda(), ps, n)
    assert "supplied (device memory)" in b.build_info
    pa, pb = plan_of(a), plan_of(b)
    assert pa[0] == pb[0], "tile descriptors differ"
    assert pa[1] == pb[1], "entry blocks differ"
    assert a.display() == b.display() and a.mapped_pixels == b.mapped_pixels and a.upload_bytes_per_frame == b.upload_bytes_per_frame
    assert np.array_equal(b.lensmap_packed(), a.lensmap_packed())   # (copied back once, on demand)
    assert a.plan_digest() == b.plan_digest()


@pytest.mark.parametrize("globe", ["cube", "fast"])
def test_plans_of_every_shipped_lens(bb, palette, torch, pair, globe):
    a, b, _ = pair
    for lens in ALL_LENSES:
        m, n = built_map(bb, palette, globe, lens, None, (200, 120, 64), rubix=True)
        assert_same_plan(torch, a, b, m, 64, n)


@pytest.mark.parametrize("globe,lens,rubix", BASELINE_4K)
def test_plans_of_the_4k_workloads(bb, palette, torch, pair, globe, lens, rubix):
    a, b, _ = pair
    m, n = built_map(bb, palette, globe, lens, ZOOM[lens], (3840, 2160, 2048), rubix, threads=0, device=0)
    assert_same_plan(torch, a, b, m, 2048, n)


@pytest.mark.parametrize("kind", RANDOM_KINDS)
def test_plans_of_random_and_adversarial_maps(torch, pair, monkeypatch, kind):
    a, b, _ = pair
    m, ps, n, max_box = random_map(kind)
    if max_box != 8192:
        monkeypatch.setenv("BLINKY_MAX_BOX", str(max_box))
    assert_same_plan(torch, a, b, m, ps, n)


def test_plans_at_the_extents(torch, pair):
    a, b, _ = pair
    rng = np.random.default_rng(2)
    # the largest plates: 6 x 6688^2 texels, indices up to 2^28 - 2^22 and beyond 2^27
    H, W, ps = 270, 480, 6688
    y, x = np.mgrid[0:H, 0:W]
    idx = (x // 80) * ps * ps + (6000 + y) * ps + 6000 + x % 80 * 8
    m = np.where(rng.random((H, W)) < 0.9, VALID | (np.uint32(TINT_NONE) << 28) | idx.astype(np.uint32), TINT_NONE << 28).astype(np.uint32)
    assert_same_plan(torch, a, b, m, ps, 6)
    # a screen 65537 pixels wide gets no plan
    m = np.full((3, 65537), TINT_NONE << 28, np.uint32)
    m[1, ::7] = VALID | (np.uint32(TINT_NONE) << 28) | np.arange(0, 65537, 7, dtype=np.uint32) % 4096
    assert_same_plan(torch, a, b, m, 64, 1)
    assert b.tile_plan()[0].size == 0


def warp_all(torch, fe, d_faces, nframes, ps, table, tables):
    """every warp configuration the map feeds; {name: (output, last_kernel)}"""
    W, H = fe.width, fe.height
    out = {}

    def run(name, fn):
        fn()
        torch.cuda.synchronize()
        out[name] = fn.result.cpu().numpy(), fe.last_kernel

    fstride = 6 * ps * ps

    def dense(rgba, kernel):
        def f():
            f.result = torch.zeros((nframes, H, W * (4 if rgba else 1)), dtype=torch.uint8, device="cuda")
            fe.set_kernel(1 if kernel == "K1" else 0)
            fe.warp(d_faces, f.result, nframes=nframes, face_stride=fstride, rgba=rgba)
            fe.set_kernel(0)
        return f

    def view(rgba, keep, x0, with_tables=False):
        def f():
            bpp = 4 if rgba else 1
            rowbytes = -(-(x0 + W + 5) * bpp // 16) * 16
            f.result = torch.full((nframes, H + 3, rowbytes), 0x5A, dtype=torch.uint8, device="cuda")
            fe.warp_view(d_faces, f.result, x0=x0, y0=2, nframes=nframes, keep_unmapped=keep, rgba=rgba, face_stride=fstride,
                         tables=tables if with_tables else None)
        return f

    fe.set_rgba_table(table)
    for rgba in (False, True):
        for kernel in ("ring", "K1"):
            run(f"dense-{kernel}-{rgba}", dense(rgba, kernel))
        for keep in (False, True):
            run(f"view-{rgba}-{keep}", view(rgba, keep, 8))
            run(f"K0-{rgba}-{keep}", view(rgba, keep, 5))
    run("tables", view(True, False, 8, True))
    return out


@pytest.mark.parametrize("nframes", [1, 5, 16])
def test_warps_equal_the_host_supplied_map(bb, palette, torch, pair, nframes):
    a, b, b3 = pair
    W, H, ps = 400, 226, 192
    m, n = built_map(bb, palette, "cube", "quincuncial", "f_cover", (W, H, ps), rubix=True)
    rng = np.random.default_rng(nframes)
    faces = rng.integers(0, 256, (nframes, 6, ps, ps), dtype=np.uint8)
    d_faces = torch.from_numpy(faces).cuda()
    table = rng.integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32)
    tables = torch.from_numpy(rng.integers(0, 2**31, (nframes, 256), dtype=np.int64).astype(np.int32)).cuda()
    bg = bb.synthetic_background(W, H)
    outs = []
    for fe, dev in ((a, False), (b, True), (b3, True)):
        fe.set_rubix(True)
        fe.set_lensmap(torch.from_numpy(m.view(np.int32)).cuda() if dev else m, ps, n)
        fe.set_background(bg)
        outs.append(warp_all(torch, fe, d_faces, nframes, ps, table, tables))
    for name, (want, kernel) in outs[0].items():
        for got, got_kernel in (outs[1][name], outs[2][name]):
            assert np.array_equal(got, want), name
    for name, (_, kernel) in outs[0].items():
        want_kernel = "K1" if "K1" in name else "K0" if name.startswith("K0") else "ring"
        assert KERNEL[want_kernel] in kernel, (name, kernel)
    assert any(KERNEL["K3"] in k for _, k in outs[2].values()), "the serial-gather context launched K3"
    # warp_host: the plate rectangles and row spans the host kept
    host_faces = faces.reshape(nframes, -1)
    for keep in (False, True):
        dst = np.full((nframes, H + 4, W + 9), 0x33, np.uint8)
        want = a.warp_host(host_faces, dst.copy(), keep_unmapped=keep, x0=9, y0=4, nframes=nframes, face_stride=6 * ps * ps)
        got = b.warp_host(host_faces, dst.copy(), keep_unmapped=keep, x0=9, y0=4, nframes=nframes, face_stride=6 * ps * ps)
        assert np.array_equal(got, want), keep


def test_atlas_face_layout(bb, palette, torch, pair):
    a, b, _ = pair
    W, H, ps = 320, 200, 128
    m, n = built_map(bb, palette, "cube", "panini", "f_fov 180", (W, H, ps))
    rowbytes, origins = 3 * ps + 32, [(0, 0), (ps, 0), (2 * ps, 0), (0, ps), (ps, ps), (2 * ps, ps)]
    surf = np.random.default_rng(4).integers(0, 256, (2, 2 * ps + 8, rowbytes), dtype=np.uint8)
    d_surf = torch.from_numpy(surf).cuda()
    outs = []
    for fe, src in ((a, m), (b, torch.from_numpy(m.view(np.int32)).cuda())):
        fe.set_lensmap(src, ps, n)
        fe.set_face_layout(rowbytes, origins)
        out = torch.zeros((2, H, W), dtype=torch.uint8, device="cuda")
        fe.warp(d_surf, out, nframes=2)
        torch.cuda.synchronize()
        outs.append((out.cpu().numpy(), fe.last_kernel))
    assert np.array_equal(outs[0][0], outs[1][0]) and KERNEL["ring"] in outs[1][1]


def test_the_map_is_read_in_stream_order(bb, palette, torch, cuda_device):
    W, H, ps = 256, 160, 64
    m, n = built_map(bb, palette, "cube", "fisheye1", "f_contain", (W, H, ps))
    fe = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        side = torch.cuda.Stream()
        d_map = torch.zeros((H, W), dtype=torch.int32, device="cuda")
        src = torch.from_numpy(m.view(np.int32)).cuda()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(100_000_000)   # the map is written well after the call is made
            d_map.copy_(src)
            fe.set_lensmap(d_map, ps, n, stream=side.cuda_stream)
        assert np.array_equal(fe.lensmap_packed(), m)
    finally:
        fe.close()


def test_an_animated_map_written_by_a_torch_kernel(bb, palette, torch, cuda_device):
    """a zoom step per frame computed on the GPU, set, then warped: each frame is the host-supplied map's warp"""
    W, H, ps = 320, 192, 128
    fe = bb.Fisheye(device=cuda_device, palette=palette)
    ref = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        y, x = torch.meshgrid(torch.arange(H, device="cuda"), torch.arange(W, device="cuda"), indexing="ij")
        faces = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (6, ps, ps), dtype=np.uint8)).cuda()
        for step in range(4):
            z = 0.3 + 0.1 * step
            px = ((x - W / 2) * z + ps / 2).long()
            py = ((y - H / 2) * z + ps / 2).long()
            ok = (px >= 0) & (px < ps) & (py >= 0) & (py < ps)
            e = (VALID | (TINT_NONE << 28)) + (step % 6) * ps * ps + py.clamp(0, ps - 1) * ps + px.clamp(0, ps - 1)
            v = torch.where(ok, e, torch.full_like(e, TINT_NONE << 28))
            d_map = (v - (v >= 2**31).long() * 2**32).to(torch.int32)   # the same 32 bits, as torch's int32
            fe.set_lensmap(d_map, ps, 6)
            ref.set_lensmap(d_map.cpu().numpy().view(np.uint32), ps, 6)
            outs = []
            for f in (fe, ref):
                out = torch.zeros((H, W * 4), dtype=torch.uint8, device="cuda")
                f.warp(faces, out, nframes=1, rgba=True)
                outs.append(out)
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[1]), step
    finally:
        fe.close()
        ref.close()


def test_refused_device_maps_leave_the_old_map_warping(bb, palette, torch, pair):
    a, b, _ = pair
    W, H, ps = 96, 64, 32
    m, n = built_map(bb, palette, "cube", "stereographic", "f_fov 200", (W, H, ps))
    b.set_lensmap(torch.from_numpy(m.view(np.int32)).cuda(), ps, n)
    faces = torch.from_numpy(np.random.default_rng(6).integers(0, 256, (6, ps, ps), dtype=np.uint8)).cuda()

    def warp():
        out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
        b.warp(faces, out)
        torch.cuda.synchronize()
        return out.cpu().numpy()

    before, plan, display = warp(), plan_of(b), b.display()
    lib = bb.load_library()
    for what, w, h, p, nn, bad in refusals():
        ptr = None if bad is None else torch.from_numpy(np.ascontiguousarray(bad).view(np.int32)).cuda()
        rc = lib.blinky_set_lensmap_device(b._ctx, w, h, p, nn, None if ptr is None else ptr.data_ptr(), None)
        assert rc == bb.E_INVALID, what
        assert np.array_equal(warp(), before), what
        assert plan_of(b) == plan and b.display() == display, what
    assert np.array_equal(b.lensmap_packed(), m)


def test_a_graph_captured_before_the_call_replays_the_old_map(bb, palette, torch, cuda_device):
    W, H, ps = 160, 96, 64
    m1, n = built_map(bb, palette, "cube", "panini", "f_fov 180", (W, H, ps))
    m2, _ = built_map(bb, palette, "cube", "hammer", "f_contain", (W, H, ps))
    fe = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        faces = torch.from_numpy(np.random.default_rng(8).integers(0, 256, (6, ps, ps), dtype=np.uint8)).cuda()
        fe.set_lensmap(torch.from_numpy(m1.view(np.int32)).cuda(), ps, n)
        out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
        fe.warp(faces, out)
        torch.cuda.synchronize()
        want1 = out.clone()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fe.warp(faces, out)
        fe.set_lensmap(torch.from_numpy(m2.view(np.int32)).cuda(), ps, n)
        eager = torch.zeros_like(out)
        fe.warp(faces, eager)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want1), "the replay rendered the map it captured"
        assert not torch.equal(eager, want1), "the eager warp renders the new map"
        del g
        fe.release_captures()
        fe.warp(faces, out)
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
    finally:
        fe.close()
