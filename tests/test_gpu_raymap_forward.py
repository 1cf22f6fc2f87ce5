"""Ray export of forward lenses on the GPU (blinky_get_raymap_forward_device, DESIGN §3h): the forward build's grid points
on the GPU, the interpreter's settled points, the quads rasterised and each pixel's ray from its winning quad, written in
stream order.  The field must equal the host export byte for byte: every forward-only lens on cube and fast, two lenses
with both functions, odd sizes, a 2W x 2H field and a 4K workload; the stream order, a capturing stream and the host
fallback; and the warps from an exported sinusoidal field against the numpy oracles of the ray warps."""
import re

import numpy as np
import pytest

import ray_bilinear_reference as br
import ray_reference as rr
import ray_trilinear_reference as tr
from test_gpu_ray_supersample import TABLE
from test_gpu_ray_warp import yaw
from test_raymap_forward_host_only import FORWARD_ONLY

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


def settled(fe):
    info = fe.build_info
    m = re.match(r"ray export \(forward\), device: (\d+) grid points settled", info)
    assert m, info
    return int(m.group(1))


def export_both(torch, fe, W, H, ps=0):
    """(host field, device field on the GPU); the device field starts as a sentinel so every element must be written"""
    host = fe.raymap(W, H, forward=True, platesize=ps)
    d = torch.full((H, W, 3), 12345.0, dtype=torch.float32, device="cuda")
    assert fe.raymap(W, H, out=d, forward=True, platesize=ps) is d
    return host, d


def assert_same_bytes(got, want, what=""):
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32, what
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (what, len(bad), [(tuple(i), got[tuple(i)], want[tuple(i)]) for i in bad[:4]])


@pytest.mark.parametrize("globe", ["cube", "fast"])
def test_every_forward_only_lens(torch, fe, globe):
    W, H = 320, 180
    fe.command(f"f_globe {globe}")
    for lens in FORWARD_ONLY:
        fe.command(f"f_lens {lens}")
        host, d = export_both(torch, fe, W, H)
        settled(fe)
        assert_same_bytes(d.cpu().numpy(), host, (globe, lens))


@pytest.mark.parametrize("lens,zoom", [("equirect", "f_contain"), ("hammer", "f_cover")])
def test_lenses_with_both_functions(torch, fe, lens, zoom):
    fe.command("f_globe cube")
    fe.command(f"f_lens {lens}")
    fe.command(zoom)
    host, d = export_both(torch, fe, 320, 180, 128)
    settled(fe)
    assert_same_bytes(d.cpu().numpy(), host, lens)


@pytest.mark.parametrize("W,H,ps", [(97, 61, 37), (1, 40, 16), (40, 1, 16), (640, 360, 0), (1280, 720, 360)])
def test_odd_sizes_and_a_double_size_field(torch, fe, W, H, ps):
    fe.command("f_globe trism")
    fe.command("f_lens winkel2")
    host, d = export_both(torch, fe, W, H, ps)
    settled(fe)
    assert_same_bytes(d.cpu().numpy(), host, (W, H, ps))


def test_4k_sinusoidal(torch, fe):
    W, H, ps = 3840, 2160, 2048
    fe.command("f_globe cube")
    fe.command("f_lens sinusoidal")
    fe.command("f_contain")
    host, d = export_both(torch, fe, W, H, ps)
    settled(fe)
    assert_same_bytes(d.cpu().numpy(), host)
    fe.build_lensmap(W, H, ps, threads=0)
    idx, _ = fe.lensmap()
    assert np.array_equal(np.any(host != 0, axis=2), idx >= 0)


def test_the_field_is_written_in_stream_order(torch, fe):
    W, H = 640, 360
    fe.command("f_globe cube")
    fe.command("f_lens sinusoidal")
    host = fe.raymap(W, H, forward=True)
    d = torch.zeros((H, W, 3), dtype=torch.float32, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)   # the sentinel lands well after the call is made
        d.fill_(-7.0)
        fe.raymap(W, H, out=d, stream=side.cuda_stream, forward=True)
        assert side.query(), "the call returns with the field complete"
    settled(fe)
    assert_same_bytes(d.cpu().numpy(), host)


def test_a_capturing_stream_is_refused(bb, torch, fe):
    W, H = 64, 48
    fe.command("f_globe cube")
    fe.command("f_lens sinusoidal")
    lib = bb.load_library()
    d = torch.zeros((H, W, 3), dtype=torch.float32, device="cuda")
    x = torch.ones(16, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = x * 2
        rc = lib.blinky_get_raymap_forward_device(fe._ctx, W, H, 0, d.data_ptr(), torch.cuda.current_stream().cuda_stream)
        y += 1
    assert rc == bb.E_STATE
    assert "capturing" in lib.blinky_last_error(fe._ctx).decode()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, torch.full_like(x, 3.0)), "the capture stays intact"
    assert not d.any()
    fe.raymap(W, H, out=d, forward=True)   # and the context still works
    assert_same_bytes(d.cpu().numpy(), fe.raymap(W, H, forward=True))


UNTRANSLATABLE = """
map = "lens_forward"
max_fov = 360
max_vfov = 180
lens_width = 2*pi
lens_height = pi
onload = "f_contain"
function lens_forward(x, y, z)
  local name = "plate carree"
  local lat, lon = ray_to_latlon(x, y, z)
  return lon, lat
end
"""


def test_the_host_fallback(torch, fe):
    fe.command("f_globe cube")
    fe.load_lens("carree", UNTRANSLATABLE)
    host, d = export_both(torch, fe, 320, 200)
    assert fe.build_info.startswith("ray export (forward), host ("), fe.build_info
    assert_same_bytes(d.cpu().numpy(), host)
    assert np.any(host != 0)


# ---- end to end: an exported sinusoidal field through the ray warps ---------------------------------------------------

W, H, PS = 96, 64, 97
YAWS = [0.0, 25.0, -40.0]


@pytest.fixture(scope="module")
def bshim(tmp_path_factory):
    return br.compile_shim(tmp_path_factory.mktemp("fwd_bilinear"))


@pytest.fixture(scope="module")
def tshim(tmp_path_factory):
    return tr.compile_shim(tmp_path_factory.mktemp("fwd_trilinear"))


def sinusoidal_view(torch, fe, k):
    """fe on cube with a W x H all-unmapped map of PS installed, the sinusoidal field at k*W x k*H: (field, bg, faces,
    matrices)"""
    fe.command("f_globe cube")
    fe.command("f_lens sinusoidal")
    fe.command("f_contain")
    fe.set_rgba_table(TABLE)
    field = torch.empty((k * H, k * W, 3), dtype=torch.float32, device="cuda")
    fe.raymap(k * W, k * H, out=field, forward=True, platesize=PS)
    bg = np.random.default_rng(3).integers(0, 256, W * H, dtype=np.uint8)
    fe.set_lensmap(np.full((H, W), 0x70000000, np.uint32), PS, fe.numplates)
    fe.set_background(bg)
    faces = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (len(YAWS), 6 * PS * PS), dtype=np.uint8)).cuda()
    xs = torch.from_numpy(np.stack([yaw(a) for a in YAWS])).cuda()
    return field, bg.reshape(H, W), faces, xs


@pytest.mark.parametrize("mode", ["nearest8", "nearest", "bilinear", "trilinear", "supersample2"])
def test_warps_of_an_exported_field_follow_their_oracles(bb, palette, torch, fe, bshim, tshim, mode):
    k = 2 if mode == "supersample2" else 1
    field, bg, faces, xs = sinusoidal_view(torch, fe, k)
    n, rgba = len(YAWS), mode != "nearest8"
    out = torch.zeros((n, H, W, 4) if rgba else (n, H, W), dtype=torch.uint8, device="cuda")
    filt = mode if mode in ("bilinear", "trilinear") else "nearest"
    bpp = 4 if rgba else 1
    fe.warp_rays(faces, out.data_ptr(), field, xs, rowbytes=bpp * W, screen_stride=bpp * W * H, nframes=n, rgba=rgba, filter=filt,
                 supersample=k)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    fld, fc, M = field.cpu().numpy(), faces.cpu().numpy(), xs.cpu().numpy()
    assert np.any(fld != 0) and np.any(np.all(fld == 0, axis=2)), "the field has mapped and unmapped pixels"
    if mode == "bilinear":
        g = br.BilinearGlobe(bb, palette, "cube", bshim)
    elif mode == "trilinear":
        g = tr.TrilinearGlobe(bb, palette, "cube", tshim)
    else:
        g = rr.HostGlobe(bb, palette, "cube")
    try:
        for f in range(n):
            if mode == "trilinear":
                want = g.frame(fld, M[f], fc[f], bg, PS, table=TABLE)[0]
            elif mode == "bilinear":
                want = g.frame(fld, M[f], fc[f], bg, 1, PS, table=TABLE)[0]
            else:
                want = rr.frame(g, fld, M[f], fc[f], bg, k, PS, table=TABLE if rgba else None)[0]
            want = np.asarray(want).reshape(got[f].shape)
            bad = np.argwhere(got[f] != want)
            assert bad.size == 0, (mode, f, len(bad), bad[:4].tolist())
    finally:
        g.close()
