"""The device lensmap builder's text behind the CPU shim (test_device_emulation's machinery) over the zoom and view-shape
sweep of zoom_sweep.py: every translatable lens and every forward-only lens on cube, at every zoom of the sweep, on a
97 x 61 view and the very wide 1000 x 8 and very tall 8 x 640 ones, with the host libm and with every libm result moved
by up to 3 and 3 * 2^20 ulp.  The zooms reach the lens functions' poles, domain edges and overflows (an infinite or NaN
scale included), where the error bounds' pole and range-edge rules decide.  No GPU involved."""
import ctypes
import math

import numpy as np
import pytest

from conftest import ALL_LENSES
from test_device_emulation import (GRID, RUN_FORWARD, RUN_INVERSE, ForwardPatch, FwdGeom, build_lib, fwd_lib, params_of,  # noqa: F401
                                   x86_int)
from test_transpile import FORWARD_ONLY, TRANSLATABLE, perturbed
from zoom_sweep import refused_past_the_limit, zoom_limits, zooms

SHAPES = [(97, 61, 48), (1000, 8, 48), (8, 640, 48)]
LIBMS = [0, 1, 1 << 20]   # 0 = host libm, else libm results off by up to 3 * scale ulp


def host_build(bb, host, lens, zoom, w, h, ps):
    """the interpreter's build: (error code or 0, idx, tint, display, "> maxdiff" messages, scale)"""
    host.command(f"f_lens {lens}")
    host.command(zoom)
    host.clear_log()
    try:
        host.build_lensmap(w, h, ps, threads=-1)
        code = 0
    except bb.BlinkyError as e:
        code = e.code
    idx, tint = host.lensmap()
    msgs = [int(l.split()[0]) for l in host.log.splitlines() if l.endswith("> maxdiff")]
    return code, idx, tint, host.display(), msgs, host.scale


class Libs:
    """one compiled shim per distinct kernel text (the text does not depend on the zoom, but nothing here assumes so)"""

    def __init__(self, tmp_path, run):
        self.tmp, self.run, self.cache = tmp_path, run, {}

    def get(self, src, scale):
        key = (src, scale)
        if key not in self.cache:
            self.cache[key] = build_lib(perturbed(src, scale) if scale else src, self.run, str(self.tmp / f"k{len(self.cache)}"))
        return self.cache[key]


@pytest.mark.parametrize("lens", TRANSLATABLE)
def test_emulated_inverse_build_over_the_zoom_sweep(bb, host, tmp_path, lens):
    host.set_rubixgrid(*GRID)
    host.command("f_globe cube")
    max_fov, max_vfov = zoom_limits(host, lens)
    libs = Libs(tmp_path, RUN_INVERSE)
    built = 0
    for zoom in zooms(max_fov, max_vfov):
        for w, h, ps in SHAPES:
            code, idx, tint, _, _, _ = host_build(bb, host, lens, zoom, w, h, ps)
            if refused_past_the_limit(zoom, max_fov, max_vfov):
                assert code == bb.E_ZOOM, (lens, zoom, code)
            if code:
                continue
            built += 1
            src = host.lens_source(with_kernel=True)
            p = params_of(host, w, h, ps)
            for scale in LIBMS:
                cand = np.zeros(w * h, np.uint32)
                libs.get(src, scale).run_lt_build(ctypes.byref(p), cand.ctypes.data_as(ctypes.c_void_p))
                cand = cand.reshape(h, w)
                risk = (cand & 0x20000000) != 0
                valid = (cand & 0x80000000) != 0
                ongrid = (cand & 0x40000000) != 0
                c_idx = np.where(valid, (cand & 0x0FFFFFFF).astype(np.int64), -1)
                c_tint = np.where(valid & ~ongrid, c_idx // (ps * ps), 255)
                # FisheyeHost::build_inverse_device's merge: the flagged pixels are the interpreter's
                got_idx = np.where(risk, idx, c_idx)
                got_tint = np.where(risk, tint, c_tint)
                what = (lens, zoom, (w, h, ps), scale, host.scale)
                assert np.array_equal(got_idx, idx), what + (int((got_idx != idx).sum()),)
                assert np.array_equal(got_tint, tint), what
                if scale == 0:
                    # the same libm: no decision may depend on the flags
                    assert np.array_equal(c_idx, idx) and np.array_equal(c_tint, tint), what
    assert built >= 6, (lens, built)


def grid_rays(host, ps):
    """float32 plate_uv_to_ray of every forward grid point (fisheye.c:1198-1214), [numplates * (ps+1)^2, 3]"""
    plates = host.plates()
    n1 = ps + 1
    out = np.zeros((len(plates) * n1 * n1, 3), np.float32)
    for pt in range(len(out)):
        i, j, plate = pt % n1, pt // n1 % n1, pt // n1 // n1
        f, r, u = (plates[plate][k:k + 3].astype(np.float32) for k in (0, 3, 6))
        uu = np.float32((i - 0.5) / ps - 0.5)
        vv = np.float32(-((j - 0.5) / ps - 0.5))
        ray = np.float32(plates[plate][10]) * f
        ray = ray + uu * r
        ray = ray + vv * u
        ln = np.float32(math.sqrt(float(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2])))
        if ln:
            ray = ray * (np.float32(1) / ln)
        out[pt] = ray
    return out


def screen_points(st, xy, scale, w, h):
    """uv_to_screen's (int)(x / scale + W/2), (int)(-y / scale + H/2) of every point the lens mapped, as x86 converts"""
    with np.errstate(all="ignore"):
        sx = xy[:, 0] / scale + float(w // 2)
        sy = -xy[:, 1] / scale + float(h // 2)
    return np.array([[x86_int(a), x86_int(b)] if s == 1 else [0, 0] for s, a, b in zip(st, sx, sy)], np.int64)


@pytest.mark.parametrize("lens", FORWARD_ONLY)
def test_emulated_forward_build_over_the_zoom_sweep(bb, host, fwd_lib, tmp_path, lens):
    """grid points behind the shim (each decided one equals the interpreter's screen point) -> the interpreter settles
    the undecided ones -> quads rasterised in ascending and random texel order: the serial builder's map, display flags
    and "> maxdiff" messages, at every zoom.  At f_fov 1 the points land ~10^4 pixels off the screen and nothing is drawn."""
    host.set_rubixgrid(*GRID)
    host.command("f_globe cube")
    max_fov, max_vfov = zoom_limits(host, lens)
    libs = Libs(tmp_path, RUN_FORWARD)
    ps = SHAPES[0][2]
    n1 = ps + 1
    P = host.numplates
    npts = P * n1 * n1
    rays = grid_rays(host, ps)
    # the lens at every grid point, once: the points do not depend on the zoom, only their screen positions do
    lf = [host.lens_forward(float(r[0]), float(r[1]), float(r[2])) for r in rays]
    st = np.array([s for s, _ in lf], np.int64)
    xy = np.array([v for _, v in lf], np.float64)
    assert (st >= 0).all(), lens
    ntex = P * ps * ps
    orders = [np.arange(ntex, dtype=np.uint32), np.random.default_rng(len(lens)).permutation(ntex).astype(np.uint32)]
    built = 0
    for zoom in zooms(max_fov, max_vfov):
        for w, h, _ in SHAPES:
            code, want_idx, want_tint, want_disp, want_msgs, scale = host_build(bb, host, lens, zoom, w, h, ps)
            if refused_past_the_limit(zoom, max_fov, max_vfov):
                assert code == bb.E_ZOOM, (lens, zoom, code)
            if code:
                continue
            built += 1
            want_pts = screen_points(st, xy, scale, w, h)
            src = host.lens_source(forward=True, with_kernel=True)
            p = params_of(host, w, h, ps)
            for libm in LIBMS:
                what = (lens, zoom, (w, h, ps), libm, scale)
                grid = np.zeros((npts, 2), np.int32)
                status = np.zeros(npts, np.uint8)
                undecided = np.zeros(npts, np.uint32)
                counters = np.zeros(16, np.uint32)
                libs.get(src, libm).run_lt_forward_points(
                    ctypes.byref(p), grid.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p),
                    undecided.ctypes.data_as(ctypes.c_void_p), counters.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint(npts))
                decided = status != 2
                assert int(counters[0]) == int((~decided).sum()), what
                assert np.array_equal(status[decided], st[decided]), what
                ok = decided & (st == 1)
                bad = np.nonzero(ok & (grid != want_pts).any(axis=1))[0]
                assert bad.size == 0, what + (bad.size, [(int(b), grid[b].tolist(), want_pts[b].tolist()) for b in bad[:4]])
                # the interpreter's answers for the undecided points (FisheyeHost::build_forward_device)
                und = undecided[: int(counters[0])].astype(np.int64)
                patches = (ForwardPatch * max(1, len(und)))()
                for k, pt in enumerate(und.tolist()):
                    patches[k].point, patches[k].status = pt, int(st[pt])
                    if st[pt] == 1:
                        patches[k].lx, patches[k].ly = int(want_pts[pt][0]), int(want_pts[pt][1])
                any_nil = int(counters[1] > 0 or (st[und] != 1).any())
                g = FwdGeom()
                g.width, g.height, g.ps, g.numplates = w, h, ps, P
                g.rubix_block, g.rubix_pad, g.rubix_unit_px = p.rubix_block, p.rubix_pad, p.rubix_unit_px
                for i in range(6):
                    g.plates[i] = p.plates[i]
                for order in orders:
                    gcopy, scopy = grid.copy(), status.copy()
                    idx = np.zeros(w * h, np.int32)
                    tint = np.zeros(w * h, np.uint8)
                    disp = (ctypes.c_int * 6)()
                    msgs = np.zeros((4096, 2), np.uint32)
                    nmsg = ctypes.c_uint()
                    fwd_lib.fwd_run(ctypes.byref(g), gcopy.ctypes.data_as(ctypes.c_void_p), scopy.ctypes.data_as(ctypes.c_void_p), patches,
                                    ctypes.c_uint(len(und)), any_nil, order.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint(ntex),
                                    idx.ctypes.data_as(ctypes.c_void_p), tint.ctypes.data_as(ctypes.c_void_p), disp,
                                    msgs.ctypes.data_as(ctypes.c_void_p), ctypes.byref(nmsg))
                    assert np.array_equal(idx.reshape(h, w), want_idx), what + (int((idx.reshape(h, w) != want_idx).sum()),)
                    assert np.array_equal(tint.reshape(h, w), want_tint), what
                    assert list(disp)[:P] == want_disp[:P], what
                    got_msgs = [int(v) for _, v in sorted(map(tuple, msgs[: nmsg.value].tolist()))]
                    assert got_msgs == want_msgs, what
    assert built >= 6, (lens, built)


@pytest.mark.parametrize("lens", ALL_LENSES)
def test_scale_does_not_depend_on_when_the_zoom_was_set(bb, palette, lens):
    """The zoom set right after the lens was loaded, after a build at the lens's own zoom, or after a build at another
    zoom and view: the same scale (bit for bit: inf and NaN included) and the same refusal.  A zoom set before the lens
    is loaded gives way to the lens's onload zoom."""
    w, h, ps = 97, 61, 48
    a = bb.Fisheye(device=None, palette=palette)
    b = bb.Fisheye(device=None, palette=palette)
    try:
        for fe in (a, b):
            fe.command("f_globe cube")
        max_fov, max_vfov = zoom_limits(a, lens)
        onload = a.onload
        a.build_lensmap(w, h, ps, threads=-1)
        onload_scale = a.scale
        for zoom in zooms(max_fov, max_vfov):
            results = []
            for steps in ([f"f_lens {lens}", zoom], [f"f_lens {lens}", "build", zoom], ["f_contain", f"f_lens {lens}", "f_vfov 1", "build3x2", zoom]):
                fe = b if len(results) else a
                for s in steps:
                    if s.startswith("build"):
                        try:
                            fe.build_lensmap(*((3, 2, 97) if s == "build3x2" else (w, h, ps)), threads=-1)
                        except bb.BlinkyError:
                            pass
                    else:
                        fe.command(s)
                try:
                    fe.build_lensmap(w, h, ps, threads=-1)
                    code = 0
                except bb.BlinkyError as e:
                    code = e.code
                results.append((code, np.float64(fe.scale).tobytes()))
            assert results[1:] == results[:1] * 2, (lens, zoom, results)
        # a zoom before the lens: the lens's onload replaces it
        b.command("f_fov 1")
        b.command(f"f_lens {lens}")
        assert b.onload == onload
        b.build_lensmap(w, h, ps, threads=-1)
        assert np.float64(b.scale).tobytes() == np.float64(onload_scale).tobytes(), (lens, onload)
    finally:
        a.close()
        b.close()
