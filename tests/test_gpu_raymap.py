"""Ray maps on the GPU: blinky_set_raymap_device maps a field of view rays in device memory through the current globe,
settles the pixels the device cannot decide with the interpreter, and plans the map on the GPU.  Everything must equal
the host path (blinky_set_raymap of the same rays): the map, the display flags, the tile plan byte for byte, and every
warp through it.  Covered: every inverse lens on cube and fast, 4K closed-form fields, random and adversarial rays,
globe_plate scripts with risk flags and stale plate slots, stream order, a look-around loop and CUDA graphs."""
import numpy as np
import pytest

from conftest import ALL_LENSES
from test_globe_plate_transpile import load_custom
from test_gpu_supplied_lensmap import plan_of, warp_all
from test_raymap_host_only import adversarial_rays, lens_rays

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture()
def pair(bb, palette, cuda_device):
    """(a GPU context fed host rays, one fed device rays)"""
    a = bb.Fisheye(device=cuda_device, palette=palette)
    b = bb.Fisheye(device=cuda_device, palette=palette)
    yield a, b
    a.close()
    b.close()


def settled(fe):
    info = fe.build_info
    assert info.startswith("ray map, device: "), info
    return int(info.split("device: ")[1].split(" ")[0])


def same_globe(a, b, globe):
    for fe in (a, b):
        fe.command(f"f_globe {globe}")


def assert_device_equals_host(torch, a, b, rays, ps):
    """a: host rays; b: the same rays from device memory"""
    a.set_raymap(rays, ps)
    assert a.build_info.startswith("ray map, host"), a.build_info
    b.set_raymap(torch.from_numpy(rays).cuda(), ps)
    n = settled(b)
    assert np.array_equal(b.lensmap_packed(), a.lensmap_packed()), b.build_info
    assert b.display() == a.display() and b.mapped_pixels == a.mapped_pixels and b.upload_bytes_per_frame == a.upload_bytes_per_frame
    pa, pb = plan_of(a), plan_of(b)
    assert pa[0] == pb[0], "tile descriptors differ"
    assert pa[1] == pb[1], "entry blocks differ"
    assert a.plan_digest() == b.plan_digest() and a.numplates == b.numplates
    return n


@pytest.mark.parametrize("globe", ["cube", "fast"])
def test_every_inverse_lens(bb, palette, torch, pair, globe):
    a, b = pair
    W, H, ps = 160, 100, 64
    lenses = 0
    for lens in ALL_LENSES:
        for fe in (a, b):
            fe.command(f"f_globe {globe}")
            fe.command(f"f_lens {lens}")
            fe.set_rubix(True)
        a.build_lensmap(W, H, ps, threads=1)   # the scale the rays are taken at
        rays = lens_rays(a, W, H)
        if rays is None:
            continue
        n = assert_device_equals_host(torch, a, b, rays, ps)
        if globe == "cube":
            assert n == 0, "argmax globes raise no flag"
        lenses += 1
    assert lenses >= 20


def test_every_warp_through_a_device_ray_map(bb, palette, torch, pair):
    a, b = pair
    W, H, ps = 400, 226, 192
    for fe in (a, b):
        fe.command("f_globe cube")
        fe.command("f_lens quincuncial")
        fe.command("f_cover")
    a.build_lensmap(W, H, ps, threads=1)
    rays = lens_rays(a, W, H)
    nframes = 5
    rng = np.random.default_rng(2)
    faces = rng.integers(0, 256, (nframes, 6, ps, ps), dtype=np.uint8)
    d_faces = torch.from_numpy(faces).cuda()
    table = rng.integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32)
    tables = torch.from_numpy(rng.integers(0, 2**31, (nframes, 256), dtype=np.int64).astype(np.int32)).cuda()
    bg = bb.synthetic_background(W, H)
    outs = []
    for fe, src in ((a, rays), (b, torch.from_numpy(rays).cuda())):
        fe.set_rubix(True)
        fe.set_raymap(src, ps)
        fe.set_background(bg)
        outs.append(warp_all(torch, fe, d_faces, nframes, ps, table, tables))
    for name, (want, _) in outs[0].items():
        assert np.array_equal(outs[1][name][0], want), name
    # a 3x2 atlas face layout
    rowbytes, origins = 3 * ps + 32, [(0, 0), (ps, 0), (2 * ps, 0), (0, ps), (ps, ps), (2 * ps, ps)]
    surf = torch.from_numpy(rng.integers(0, 256, (2, 2 * ps + 8, rowbytes), dtype=np.uint8)).cuda()
    got = []
    for fe in (a, b):
        fe.set_face_layout(rowbytes, origins)
        out = torch.zeros((2, H, W), dtype=torch.uint8, device="cuda")
        fe.warp(surf, out, nframes=2)
        torch.cuda.synchronize()
        got.append(out.cpu().numpy())
    assert np.array_equal(got[0], got[1])


def equirect_rays(torch, W, H, yaw=0.0):
    y, x = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float64), torch.arange(W, device="cuda", dtype=torch.float64), indexing="ij")
    lon = (x / W - 0.5) * 2 * np.pi + yaw
    lat = (0.5 - y / H) * np.pi
    return torch.stack([torch.sin(lon) * torch.cos(lat), torch.sin(lat), torch.cos(lon) * torch.cos(lat)], -1).float().contiguous()


def rectilinear_rays(torch, W, H):
    y, x = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float32), torch.arange(W, device="cuda", dtype=torch.float32), indexing="ij")
    f = W / 2 / np.tan(np.radians(50))
    return torch.stack([(x - W / 2) / f, -(y - H / 2) / f, torch.ones_like(x)], -1).contiguous()


@pytest.mark.parametrize("globe", ["cube", "trism", "fast"])
def test_4k_closed_form_fields(torch, pair, globe):
    a, b = pair
    W, H, ps = 3840, 2160, 2048
    same_globe(a, b, globe)
    for field in (equirect_rays(torch, W, H), rectilinear_rays(torch, W, H)):
        n = assert_device_equals_host(torch, a, b, field.cpu().numpy(), ps)
        if globe != "fast":
            assert n == 0, b.build_info


@pytest.mark.parametrize("globe", ["cube", "fast", "tetra"])
def test_random_and_adversarial_rays_at_1080p(torch, pair, globe):
    a, b = pair
    W, H, ps = 1920, 1080, 1024
    same_globe(a, b, globe)
    rng = np.random.default_rng(5)
    rays = rng.normal(size=(H * W, 3)).astype(np.float32)
    rays[rng.random(H * W) < 0.01] = 0
    adv = adversarial_rays(np.vstack([a.plates(), np.zeros((6 - a.numplates, 11), np.float32)]), a.numplates, ps)
    rays[: len(adv) * 50 : 50] = adv
    with np.errstate(all="ignore"):
        assert_device_equals_host(torch, a, b, rays.reshape(H, W, 3), ps)


@pytest.mark.parametrize("name", ["nan_huge", "stale", "latlon", "fractions"])
def test_globe_plate_scripts_with_risk_flags(torch, pair, name):
    """NaN and +-1e12 plates are always the interpreter's; the stale globe maps onto plate slots 2..5 the cube left"""
    a, b = pair
    W, H, ps = 320, 200, 128
    for fe in (a, b):
        load_custom(fe, name)
    rng = np.random.default_rng(8)
    rays = rng.normal(size=(H, W, 3)).astype(np.float32)
    n = assert_device_equals_host(torch, a, b, rays, ps)
    if name == "nan_huge":
        assert n > 0, b.build_info
    if name == "stale":
        assert b.numplates == 2 and (b.lensmap()[0] >= 2 * ps * ps).any()
        # and what a build of a lens returning these rays makes: the supplied-lensmap tests compare builds and maps
        b.build_lensmap(W, H, ps, threads=1)
        built = lens_rays(b, W, H)
        b.set_raymap(torch.from_numpy(built).cuda(), ps)
        dev = b.lensmap_packed().copy(), b.display()
        b.build_lensmap(W, H, ps, threads=1)
        assert np.array_equal(dev[0], b.lensmap_packed()) and dev[1] == b.display()


def test_the_rays_are_read_in_stream_order(torch, pair):
    a, b = pair
    W, H, ps = 640, 360, 256
    same_globe(a, b, "cube")
    want = equirect_rays(torch, W, H, 0.3)
    a.set_raymap(want.cpu().numpy(), ps)
    side = torch.cuda.Stream()
    d = torch.zeros_like(want)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)   # the rays are written well after the call is made
        d.copy_(equirect_rays(torch, W, H, 0.3))
        b.set_raymap(d, ps, stream=side.cuda_stream)
    assert np.array_equal(b.lensmap_packed(), a.lensmap_packed())


def test_a_look_around_loop(torch, pair):
    """a yaw per frame turns the rays on the GPU; each frame's warp equals the warp of the host ray map"""
    a, b = pair
    W, H, ps = 480, 270, 256
    same_globe(a, b, "cube")
    faces = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (6, ps, ps), dtype=np.uint8)).cuda()
    base = equirect_rays(torch, W, H)
    for step in range(6):
        c, s = np.cos(0.2 * step), np.sin(0.2 * step)
        rot = torch.tensor([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=torch.float32, device="cuda")
        rays = (base @ rot.T).contiguous()
        b.set_raymap(rays, ps)
        a.set_raymap(rays.cpu().numpy(), ps)
        outs = []
        for fe in (a, b):
            out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
            fe.warp(faces, out)
            outs.append(out)
        torch.cuda.synchronize()
        assert torch.equal(outs[0], outs[1]), step


def test_a_graph_captured_before_the_call_replays_the_old_map(torch, bb, palette, cuda_device):
    W, H, ps = 160, 96, 64
    fe = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        fe.command("f_globe cube")
        faces = torch.from_numpy(np.random.default_rng(8).integers(0, 256, (6, ps, ps), dtype=np.uint8)).cuda()
        fe.set_raymap(equirect_rays(torch, W, H), ps)
        out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
        fe.warp(faces, out)
        torch.cuda.synchronize()
        want1 = out.clone()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fe.warp(faces, out)
        fe.set_raymap(equirect_rays(torch, W, H, 1.0), ps)
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


def test_refusals_leave_the_old_map(bb, torch, pair):
    _, b = pair
    W, H, ps = 96, 64, 32
    b.command("f_globe cube")
    rays = equirect_rays(torch, W, H)
    b.set_raymap(rays, ps)
    before, plan = b.lensmap_packed().copy(), plan_of(b)
    lib = bb.load_library()
    for what, w, h, p, ptr in [("NULL", W, H, ps, None), ("misaligned", W, H, ps, rays.data_ptr() + 2), ("size", 0, H, ps, rays.data_ptr()),
                               ("platesize", W, H, 7000, rays.data_ptr())]:
        assert lib.blinky_set_raymap_device(b._ctx, w, h, p, ptr, None) == bb.E_INVALID, what
        assert np.array_equal(b.lensmap_packed(), before) and plan_of(b) == plan, what
