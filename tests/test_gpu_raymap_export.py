"""Ray export on the GPU: blinky_get_raymap_device evaluates the translated lens_inverse at every pixel of a build,
lets the interpreter settle the risk-flagged pixels, and writes the field into device memory in stream order.  The
field must equal the host export (NaN as NaN), and set_raymap_device of it must install the build's map and tile plan.
Covered: every translatable inverse lens on cube and fast, the 4K workloads, stream order, the host fallbacks
(untranslatable lens, flagged-list overflow), a capturing stream, and a look-around loop that starts from a Lua lens."""
import ctypes
import re

import numpy as np
import pytest

from test_gpu_supplied_lensmap import plan_of
from test_raymap_export_host_only import assert_same_rays
from test_transpile import TRANSLATABLE

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
    assert info.startswith("ray export, device: "), info
    return int(info.split("device: ")[1].split(" ")[0])


def export_both(torch, fe, W, H):
    """(host field, device field as numpy); the device field starts as a sentinel so every element must be written"""
    with np.errstate(all="ignore"):
        host = fe.raymap(W, H)
    d = torch.full((H, W, 3), 12345.0, dtype=torch.float32, device="cuda")
    assert fe.raymap(W, H, out=d) is d
    return host, d


def assert_round_trip_equals_the_build(torch, fe, d_rays, W, H, ps):
    fe.build_lensmap(W, H, ps, threads=0)
    info = fe.build_info
    want, want_plan, want_display = fe.lensmap_packed().copy(), plan_of(fe), fe.display()
    fe.set_raymap(d_rays, ps)
    assert fe.build_info.startswith("ray map, device"), fe.build_info
    assert np.array_equal(fe.lensmap_packed(), want)
    assert plan_of(fe) == want_plan and fe.display() == want_display
    return info


@pytest.mark.parametrize("globe", ["cube", "fast"])
def test_every_translatable_inverse_lens(torch, fe, globe):
    W, H, ps = 640, 480, 256
    fe.command(f"f_globe {globe}")
    checked = 0
    for lens in TRANSLATABLE:
        fe.command(f"f_lens {lens}")
        if fe.map_type != 1:
            continue
        host, d = export_both(torch, fe, W, H)
        n = settled(fe)
        assert_same_rays(d.cpu().numpy(), host, lens)
        info = assert_round_trip_equals_the_build(torch, fe, d, W, H, ps)
        if globe == "cube":   # an argmax globe flags nothing: every build flag comes from the lens
            m = re.match(r"device: (\d+) of \d+ pixels re-evaluated", info)
            assert m, info
            assert n == int(m.group(1)), (lens, n, info)
        checked += 1
    assert checked >= 15, checked


WORKLOADS = [("panini", "f_fov 180"), ("stereographic", "f_fov 180"), ("equirect", "f_contain"), ("hammer", "f_contain"),
             ("fisheye1", "f_contain"), ("quincuncial", "f_cover")]


@pytest.mark.parametrize("lens,zoom", WORKLOADS)
def test_4k_workloads(torch, fe, lens, zoom):
    W, H, ps = 3840, 2160, 2048
    fe.command("f_globe cube")
    fe.command(f"f_lens {lens}")
    fe.command(zoom)
    host, d = export_both(torch, fe, W, H)
    settled(fe)
    assert_same_rays(d.cpu().numpy(), host, lens)
    assert_round_trip_equals_the_build(torch, fe, d, W, H, ps)


def test_the_field_is_written_in_stream_order(torch, fe):
    W, H = 640, 360
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    host = fe.raymap(W, H)
    d = torch.zeros((H, W, 3), dtype=torch.float32, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)   # the sentinel lands well after the call is made
        d.fill_(-7.0)
        fe.raymap(W, H, out=d, stream=side.cuda_stream)
        assert side.query(), "the call returns with the field complete"
    settled(fe)
    assert_same_rays(d.cpu().numpy(), host)


MIDPOINT_LENS = """
lens_width = 2
lens_height = 2
function lens_inverse(x, y)
  local a = math.cos(0*x) + 5.9604644775390625e-08
  return a, a + 0*y, a
end
"""


def test_the_host_fallbacks(torch, fe):
    # a lens outside the translatable subset
    fe.command("f_globe cube")
    fe.command("f_lens debug")
    host, d = export_both(torch, fe, 320, 200)
    assert fe.build_info.startswith("ray export, host ("), fe.build_info
    assert_same_rays(d.cpu().numpy(), host)
    # every pixel on a float32 rounding midpoint through a libm call: the flagged list overflows at 1920x1080
    fe.load_lens("midpoint", MIDPOINT_LENS)
    fe.command("f_contain")
    host, d = export_both(torch, fe, 1920, 1080)
    assert fe.build_info.startswith("ray export, host (too many pixels need the interpreter"), fe.build_info
    assert_same_rays(d.cpu().numpy(), host)
    # below the list's capacity the same lens is settled pixel by pixel
    host, d = export_both(torch, fe, 640, 480)
    assert settled(fe) == 640 * 480
    assert_same_rays(d.cpu().numpy(), host)


def test_a_capturing_stream_is_refused(bb, torch, fe):
    W, H = 64, 48
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    lib = bb.load_library()
    d = torch.zeros((H, W, 3), dtype=torch.float32, device="cuda")
    x = torch.ones(16, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = x * 2
        rc = lib.blinky_get_raymap_device(fe._ctx, W, H, d.data_ptr(), torch.cuda.current_stream().cuda_stream)
        y += 1
    assert rc == bb.E_STATE
    assert "capturing" in lib.blinky_last_error(fe._ctx).decode()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, torch.full_like(x, 3.0)), "the capture stays intact"
    assert not d.any()
    fe.raymap(W, H, out=d)   # and the context still works
    assert_same_rays(d.cpu().numpy(), fe.raymap(W, H))


def test_a_look_around_loop_from_a_lua_lens(bb, palette, torch, cuda_device):
    """panini's rays, exported once and turned by a yaw per frame in torch; each frame's device ray map warps like the
    host ray map of the same rays, and yaw 0 warps like the build"""
    W, H, ps = 480, 270, 256
    a = bb.Fisheye(device=cuda_device, palette=palette)
    b = bb.Fisheye(device=cuda_device, palette=palette)
    try:
        for f in (a, b):
            f.command("f_globe cube")
            f.command("f_lens panini")
            f.command("f_fov 180")
        base = torch.empty((H, W, 3), dtype=torch.float32, device="cuda")
        b.raymap(W, H, out=base)
        faces = torch.from_numpy(np.random.default_rng(2).integers(0, 256, (6, ps, ps), dtype=np.uint8)).cuda()

        def warp(f):
            out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
            f.warp(faces, out)
            torch.cuda.synchronize()
            return out

        a.build_lensmap(W, H, ps, threads=0)
        built = warp(a)
        for step in range(6):
            if step == 0:
                rays = base
            else:
                c, s = np.cos(0.3 * step), np.sin(0.3 * step)
                rot = torch.tensor([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=torch.float32, device="cuda")
                rays = (base @ rot.T).contiguous()
            b.set_raymap(rays, ps)
            a.set_raymap(rays.cpu().numpy(), ps)
            got = warp(b)
            assert torch.equal(got, warp(a)), step
            if step == 0:
                assert torch.equal(got, built)
            else:
                assert not torch.equal(got, built), step
    finally:
        a.close()
        b.close()
