"""Ray export (blinky_get_raymap) on host-only contexts: the view rays a build evaluates, in the layout set_raymap reads,
so that set_raymap of an export installs the build's lensmap.  Every inverse lens on every globe in the golden order,
against the per-pixel lens_inverse of test_raymap_host_only.py and the compiled reference's fixtures; the zoom modes
before any build; the state an export leaves alone; refusals; the ray-export kernel's text behind the CPU shim of
test_device_emulation.py, with the host libm and a perturbed one.  The GPU path is tests/test_gpu_raymap_export.py."""
import ctypes
import json
import os

import numpy as np
import pytest

from conftest import ALL_LENSES
from test_device_emulation import GRID, build_lib, params_of
from test_raymap_host_only import lens_rays, map_state
from test_supplied_lensmap_host_only import assert_same_state, state
from test_transpile import TRANSLATABLE, perturbed

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def assert_same_rays(got, want, what=""):
    """bit for bit, the sign of zero included; NaN components compare as NaN (payloads and signs may differ)"""
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32, what
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), (what, int((gn != wn).sum()))
    g = np.where(gn, np.float32(0), got).view(np.uint32)
    w = np.where(wn, np.float32(0), want).view(np.uint32)
    bad = np.argwhere(g != w)
    assert bad.size == 0, (what, len(bad), [(tuple(i), got[tuple(i)], want[tuple(i)]) for i in bad[:4]])


def test_every_inverse_lens_on_every_globe_round_trips_to_the_build_and_the_reference(host):
    lm = np.load(os.path.join(G, "lensmaps_small.npz"))
    meta = json.load(open(os.path.join(G, "meta_small.json")))
    W, H, PS = 128, 96, 48
    rays_of = {}   # the per-pixel interpreter runs once per lens: only debug's rays depend on the globe (read at load)
    checked = 0
    for key in sorted(meta):   # the golden order: later globes see the plate slots earlier ones left
        g, l = key.split("__")
        host.command(f"f_globe {g}")
        host.command(f"f_lens {l}")
        host.build_lensmap(W, H, PS, threads=1)
        want = map_state(host)
        lk = key if l == "debug" else l
        if lk not in rays_of:
            rays_of[lk] = lens_rays(host, W, H), host.scale
        ref_rays, scale = rays_of[lk]
        if ref_rays is None:
            with pytest.raises(Exception, match="no per-pixel ray"):
                host.raymap(W, H)
            continue
        assert host.scale == scale
        with np.errstate(all="ignore"):
            rays = host.raymap(W, H)
        assert host.build_info.startswith("ray export, host"), host.build_info
        assert_same_rays(rays, ref_rays, key)
        host.set_raymap(rays, PS)
        got = map_state(host)
        assert_same_state(want, got)
        assert np.array_equal(got["idx"], lm[key + "__idx"]), key
        assert np.array_equal(got["tint"], lm[key + "__tint"]), key
        assert got["display"] == meta[key]["display"], key
        checked += 1
    assert checked >= 40, checked


@pytest.mark.parametrize("globe", ["cube", "trism", "fast"])
def test_rubix_grids_and_odd_sizes_round_trip(host, globe):
    host.set_rubix(True)
    host.set_rubixgrid(4, 3.0, 2.0)
    host.command(f"f_globe {globe}")
    for lens in ALL_LENSES[1::3]:
        host.command(f"f_lens {lens}")
        host.build_lensmap(97, 63, 37, threads=1)
        if host.map_type != 1:
            continue
        want = map_state(host)
        host.set_raymap(host.raymap(97, 63), 37)
        assert_same_state(want, map_state(host))


ZOOMS = ["f_fov 180", "f_fov 1000", "f_vfov 90", "f_cover", "f_contain"]


@pytest.mark.parametrize("zoom", ZOOMS)
@pytest.mark.parametrize("lens", ["panini", "fisheye1", "quincuncial", "eckert4", "stereographic", "equirect"])
def test_an_export_before_any_build_takes_the_build_scale(bb, palette, lens, zoom):
    W, H = 120, 72
    fe = bb.Fisheye(device=None, palette=palette)
    try:
        fe.command(f"f_lens {lens}")
        fe.command(zoom)
        scale0 = fe.scale
        fe.clear_log()
        try:
            rays = fe.raymap(W, H)
        except bb.BlinkyError as e:
            assert e.code == bb.E_ZOOM, str(e)
            msg = fe.log
            assert msg and fe.scale == scale0
            fe.command("f_globe cube")
            fe.clear_log()
            with pytest.raises(bb.BlinkyError) as b:
                fe.build_lensmap(W, H, 48, threads=1)
            assert b.value.code == bb.E_ZOOM
            assert msg in fe.log, (msg, fe.log)   # the build's console message
            return
        assert fe.scale == scale0, "an export leaves blinky_scale alone"
        assert fe.build_info.startswith("ray export, host")
        fe.command("f_globe cube")
        fe.build_lensmap(W, H, 48, threads=1)
        assert_same_rays(rays, lens_rays(fe, W, H), (lens, zoom))
        # another size after a build: that size's scale, and the build's scale stays
        scale = fe.scale
        small = fe.raymap(W // 2 + 1, H // 2 + 1)
        assert fe.scale == scale
        fe.build_lensmap(W // 2 + 1, H // 2 + 1, 32, threads=1)
        assert_same_rays(small, lens_rays(fe, W // 2 + 1, H // 2 + 1), (lens, zoom, "small"))
    finally:
        fe.close()


def test_an_export_changes_nothing(host):
    W, H, ps = 96, 64, 32
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.command("f_fov 180")
    host.build_lensmap(W, H, ps, threads=1)
    before = state(host)
    scale = host.scale
    host.raymap(200, 100)
    assert_same_state(before, state(host))
    assert host.scale == scale and (host.width, host.height, host.platesize) == (W, H, ps)
    assert not host.needs_rebuild(W, H, ps)
    # pending changes stay pending
    host.command("f_lens hammer")
    host.command("f_globe trism")
    host.command("f_fov 170")
    assert host.needs_rebuild(W, H, ps)
    host.raymap(W, H)
    assert host.needs_rebuild(W, H, ps)
    assert_same_state(before, state(host))
    assert host.scale == scale


def test_no_globe_is_needed(bb, palette):
    fe = bb.Fisheye(device=None, palette=palette)
    try:
        fe.command("f_lens stereographic")
        fe.command("f_fov 200")
        rays = fe.raymap(40, 30)
        assert not fe.globe_valid
        fe.command("f_globe cube")
        fe.build_lensmap(40, 30, 16, threads=1)
        assert_same_rays(rays, lens_rays(fe, 40, 30))
    finally:
        fe.close()


FORWARD_OF_INVERSE = """
max_fov = 360
max_vfov = 180
map = "lens_forward"
function lens_inverse(x, y) return x, y, 1 end
function lens_forward(x, y, z) return x / z, y / z end
"""


def test_refusals(bb, host):
    lib = bb.load_library()
    buf = np.zeros(3 * 64 + 1, np.float32)
    assert lib.blinky_get_raymap(host._ctx, 8, 8, buf.ctypes.data) == bb.E_STATE, "no lens"
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.command("f_fov 180")
    host.build_lensmap(32, 24, 16, threads=1)
    before = state(host)
    info = host.build_info
    for what, w, h, ptr in [("NULL rays", 8, 8, None), ("misaligned", 8, 8, buf.ctypes.data + 2), ("width 0", 0, 8, buf.ctypes.data),
                            ("height < 0", 8, -1, buf.ctypes.data)]:
        assert lib.blinky_get_raymap(host._ctx, w, h, ptr) == bb.E_INVALID, what
        assert_same_state(before, state(host))
        assert host.build_info == info
    assert lib.blinky_get_raymap_device(host._ctx, 8, 8, buf.ctypes.data, None) == bb.E_NODEVICE
    # forward-only lenses and map = "lens_forward" have no per-pixel ray
    forward_only = 0
    for lens in ALL_LENSES:
        host.command(f"f_lens {lens}")
        if host.map_type == 2:
            assert lib.blinky_get_raymap(host._ctx, 8, 8, buf.ctypes.data) == bb.E_STATE, lens
            forward_only += 1
    assert forward_only
    host.load_lens("fwd", FORWARD_OF_INVERSE)
    assert lib.blinky_get_raymap(host._ctx, 8, 8, buf.ctypes.data) == bb.E_STATE
    assert "lens_forward" in lib.blinky_last_error(host._ctx).decode()
    # a raising lens and a lens returning two values: E_SCRIPT with call_inverse's messages
    for src, msg in [("max_fov = 360\nmax_vfov = 180\nlens_width = 2\nfunction lens_inverse(x, y) if x > 0.5 then error('boom') end return x, y, 1 end",
                      "boom"),
                     ("lens_width = 2\nfunction lens_inverse(x, y) return x, y end", "instead of 3")]:
        host.load_lens("bad", src)
        host.command("f_contain")
        host.clear_log()
        assert lib.blinky_get_raymap(host._ctx, 64, 1, buf.ctypes.data) == bb.E_SCRIPT
        assert msg in host.log, host.log
        assert_same_state(before, state(host))
    assert host.build_info == info


# ---- the ray-export kernel's text behind the CPU shim ------------------------------------------------------------------

RUN_RAYS = r"""
extern "C" void run_lt_rays(const LtParams *P, float *rays, unsigned *flagged, unsigned *nflagged, unsigned cap) {
    blockDim.x = 128; blockDim.y = blockDim.z = 1;
    for (unsigned by = 0; by < (unsigned)P->height; ++by)
        for (unsigned bx = 0; bx * 128 < (unsigned)P->width; ++bx)
            for (unsigned t = 0; t < 128; ++t) {
                blockIdx.x = bx; blockIdx.y = by; blockIdx.z = 0; threadIdx.x = t;
                lt_rays(*P, rays, flagged, nflagged, cap);
            }
}
"""


@pytest.mark.parametrize("scale", [0, 1 << 20])   # 0 = host libm, else libm results off by up to 3*scale ulp
@pytest.mark.parametrize("lens", TRANSLATABLE)
def test_emulated_rays_kernel_equals_the_host_path(host, tmp_path, lens, scale):
    w, h, ps = 96, 64, 48
    host.set_rubixgrid(*GRID)
    host.command("f_globe tetra")   # (the plates do not enter the unit)
    host.command(f"f_lens {lens}")
    host.build_lensmap(w, h, ps, threads=1)   # the scale, for params_of
    if host.map_type != 1:
        pytest.skip("forward lens")
    with np.errstate(all="ignore"):
        want = host.raymap(w, h).reshape(-1, 3)
    src = host.lens_source(rays=True)
    assert src.startswith(host.lens_source()) and "lt_rays" in src and "LT_HAS_GLOBE_PLATE 1" not in src
    if scale:
        src = perturbed(src, scale)
    lib = build_lib(src, RUN_RAYS, str(tmp_path / f"rays_{lens}_{scale}"))
    p = params_of(host, w, h, ps)
    got = np.full((h * w, 3), np.float32(12345.0))
    flagged = np.zeros(h * w, np.uint32)
    n = ctypes.c_uint(0)
    lib.run_lt_rays(ctypes.byref(p), got.ctypes.data_as(ctypes.c_void_p), flagged.ctypes.data_as(ctypes.c_void_p), ctypes.byref(n),
                    ctypes.c_uint(h * w))
    flagged = flagged[: n.value]
    keep = np.ones(h * w, bool)
    keep[flagged] = False
    assert_same_rays(got[keep], want[keep], (lens, scale, "unflagged"))
    got[flagged] = want[flagged]   # the host's rays for the flagged pixels
    assert_same_rays(got, want, (lens, scale, "merged"))


def test_rays_source_flavour(bb, host):
    host.command("f_lens panini")
    cuda = host.lens_source(cuda=True, rays=True)
    assert cuda.startswith(host.lens_source(cuda=True)) and "lt_rays" in cuda and "#define LT_FN static __device__" in cuda
    host.command("f_globe fast")   # a globe_plate script does not enter the unit; bits 1 to 4 are ignored
    assert host.lens_source(cuda=True, rays=True) == cuda
    assert host.lens_source(cuda=True, rays=True, forward=True, with_kernel=True, globe_plate=True, raymap=True) == cuda
    # the build kernel's pixel text is shared word for word
    build = host.lens_source(cuda=True, with_kernel=True)
    head = build[build.index("    const int lx = "): build.index("        float len = ray[0]")]
    assert head in cuda
    host.command("f_lens debug")
    with pytest.raises(bb.BlinkyError):
        host.lens_source(rays=True)
