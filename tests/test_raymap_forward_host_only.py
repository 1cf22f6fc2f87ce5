"""Ray export of forward lenses (blinky_get_raymap_forward, DESIGN §3h) without a GPU.

- The per-pixel rule of forward_raster.h (fwd_quad_st, fwd_quad_ray), compiled with g++ -ffp-contract=off, against an
  independent numpy restatement on synthetic quads: points, lines, zero-area, convex, concave and bow-tie quads, pixels
  on vertices and edges and outside both triangles, corners wrapped at INT_MIN / INT_MAX.
- The device pipeline on the CPU: grid points from the NVRTC text behind the shim of test_device_emulation.py, the
  interpreter's undecided points and texel owners, fwd_stale_chain, fwd_raster_texel in shuffled orders and
  fwd_ray_pixel, bit for bit against the host export.
- Mapped-ness against the forward build, each ray inside its winning texel's quad rectangle, the round trip through
  lens_forward, the angle to the inverse export for lenses with both functions, refusals and the state an export
  leaves alone.  The GPU path is tests/test_gpu_raymap_forward.py."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

from test_device_emulation import GRID, HOLES, RUN_FORWARD, FwdGeom, ForwardPatch, build_lib, params_of, x86_int
from test_supplied_lensmap_host_only import assert_same_state, state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the shipped lenses with lens_forward only
FORWARD_ONLY = ["sinusoidal", "kavrayskiy7", "wagner6", "larrivee", "eckert1", "eckert5", "winkel1", "winkel2", "polyconic", "gins8"]
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1

HARNESS = r"""
#include <vector>
#include <cstring>
#include "forward_raster.h"
using namespace blinky;
extern "C" int sizeof_geom() { return (int)sizeof(FwdGeom); }
extern "C" void quad_st(const int *cx, const int *cy, int n, const int *px, const int *py, double *s, double *t) {
    for (int i = 0; i < n; ++i) fwd_quad_st(cx + 4 * i, cy + 4 * i, px[i], py[i], s + i, t + i);
}
extern "C" void quad_ray(const FwdGeom *g, int plate, int ps, int tx, int ty, const int *cx, const int *cy, int n, const int *px, const int *py,
                         float *rays) {
    for (int i = 0; i < n; ++i) fwd_quad_ray(g->plates[plate], ps, tx, ty, cx + 4 * i, cy + 4 * i, px[i], py[i], rays + 3 * i);
}
// the device's steps 2-3 and the ray kernel: patches -> stale replay -> every texel in the order given -> each pixel's ray
extern "C" void run_rays(const FwdGeom *g, FwdPoint *grid, unsigned char *status, const ForwardPatch *patches, unsigned npatch, int any_nil,
                         const unsigned char *owner, const unsigned *order, unsigned ntexels, float *rays) {
    for (unsigned k = 0; k < npatch; ++k) fwd_apply_patch(grid, status, patches[k]);
    if (any_nil)
        for (int t = 2 * (g->ps + 1) - 1; t >= 0; --t) fwd_stale_chain(grid, status, g->ps, g->numplates, t);
    const size_t npix = (size_t)g->width * g->height;
    std::vector<unsigned> keys(2 * npix, 0u);
    unsigned counters[16];
    memset(counters, 0, sizeof counters);
    std::vector<FwdMessage> messages(kFwdMessageCap);
    FwdOut o{keys.data(), keys.data() + npix, counters, messages.data()};
    for (unsigned k = 0; k < ntexels; ++k) {
        const unsigned t = order[k];
        fwd_raster_texel(*g, grid, o, t / g->ps / g->ps, t / g->ps % g->ps, t % g->ps, owner);
    }
    for (size_t at = 0; at < npix; ++at) fwd_ray_pixel(*g, grid, keys[at], (int)(at % g->width), (int)(at / g->width), rays + 3 * at);
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("fwd_rays")
    src = d / "harness.cpp"
    src.write_text(HARNESS)
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(ROOT, "blinky_b200", "csrc"),
                        "-o", str(d / "harness.so"), str(src)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:3000]
    so = ctypes.CDLL(str(d / "harness.so"))
    assert so.sizeof_geom() == ctypes.sizeof(FwdGeom)
    return so


# ---- the rule, restated ----------------------------------------------------------------------------------------------

def rule_st(cx, cy, X, Y):
    """(s, t) of pixel (X, Y) in the quad cx, cy = {tl, tr, br, bl}: Python integers, then one float64 division each"""
    if any(abs(cx[i] - cx[0]) > 20 or abs(cy[i] - cy[0]) > 20 for i in range(4)):
        return 0.5, 0.5
    q = [(2 * (cx[i] - cx[0]), 2 * (cy[i] - cy[0])) for i in range(4)]
    p = (2 * (X - cx[0]) - 1, 2 * (Y - cy[0]) - 1)

    def cross(a, b):
        return a[0] * b[1] - a[1] * b[0]

    first = None
    for name, (v1, v2) in (("A", (q[1], q[2])), ("B", (q[2], q[3]))):
        area = cross(v1, v2)
        if area == 0:
            continue
        l1, l2 = cross(p, v2), cross(v1, p)   # the areas opposite V1 and V2, i.e. their weights times area
        l0 = area - l1 - l2
        inside = all(a >= 0 for a in (l0, l1, l2)) if area > 0 else all(a <= 0 for a in (l0, l1, l2))
        s, t = (l1 + l2, l2) if name == "A" else (l1, l1 + l2)
        st = (float(np.float64(s) / np.float64(area)), float(np.float64(t) / np.float64(area)))
        if inside:
            return st
        if first is None:
            first = st
    if first is None:
        return 0.5, 0.5
    return tuple(min(1.0, max(0.0, v)) for v in first)


def rule_ray(plate_row, ps, tx, ty, s, t):
    """plate_uv_to_ray of the plate point ((tx - 1/2 + s) / ps, (ty - 1/2 + t) / ps) in float32 (fisheye.c:1198-1214)"""
    u = ((tx - 0.5) + s) / ps
    v = ((ty - 0.5) + t) / ps
    f, r, up = (np.asarray(plate_row[k:k + 3], np.float32) for k in (0, 3, 6))
    uu, vv = np.float32(u - 0.5), np.float32(-(v - 0.5))
    ray = np.zeros(3, np.float32) + np.float32(plate_row[10]) * f
    ray = ray + uu * r
    ray = ray + vv * up
    ln = np.float32(math.sqrt(float(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2])))
    if ln:
        ray = ray * (np.float32(1) / ln)
    return ray


def synthetic_quads():
    """(cx, cy, X, Y) cases: every named shape with pixels on its vertices, edges, inside and outside, plus random quads"""
    shapes = {
        "point": [(5, 5)] * 4,
        "horizontal line": [(3, 7), (9, 7), (9, 7), (3, 7)],
        "vertical line": [(4, 2), (4, 2), (4, 9), (4, 9)],
        "diagonal line": [(0, 0), (3, 3), (6, 6), (9, 9)],
        "collapsed top": [(5, 5), (5, 5), (9, 12), (1, 12)],
        "collapsed right": [(0, 0), (8, 4), (8, 4), (0, 9)],
        "square": [(10, 10), (14, 10), (14, 14), (10, 14)],
        "skewed": [(10, 10), (16, 12), (15, 19), (8, 15)],
        "counter-clockwise": [(10, 10), (10, 15), (16, 15), (16, 10)],
        "concave": [(0, 0), (10, 4), (4, 4), (4, 10)],
        "bow-tie": [(0, 0), (8, 0), (0, 8), (8, 8)],
        "twisted": [(0, 0), (8, 8), (8, 0), (0, 8)],
        "at the limit": [(0, 0), (20, 0), (20, 20), (-20, 20)],
        "past the limit": [(0, 0), (21, 0), (21, 21), (0, 21)],
        "wrapped": [(INT_MAX, 3), (INT_MIN, 3), (INT_MIN, 4), (INT_MAX, 4)],
        "wrapped rows": [(3, INT_MAX), (4, INT_MAX), (4, INT_MIN), (3, INT_MIN)],
    }
    cases = []
    for name, c in shapes.items():
        cx, cy = [p[0] for p in c], [p[1] for p in c]
        if name.startswith("wrapped"):
            pts = [(3, 4), (4, 3), (0, 0)]
        else:
            x0, x1, y0, y1 = min(cx) - 2, max(cx) + 2, min(cy) - 2, max(cy) + 2
            pts = [(x, y) for y in range(y0, y1 + 1) for x in range(x0, x1 + 1)]
        cases += [(cx, cy, x, y) for x, y in pts]
    rng = np.random.default_rng(11)
    for _ in range(3000):
        base = rng.integers(-50, 3000, 2)
        off = rng.integers(-6, 7, (4, 2))
        off[0] = 0
        c = base + off
        x, y = c[0] + rng.integers(-7, 8, 2)
        cases.append(([int(v) for v in c[:, 0]], [int(v) for v in c[:, 1]], int(x), int(y)))
    return cases


def test_the_quad_position_follows_the_rule(lib):
    cases = synthetic_quads()
    n = len(cases)
    cx = np.array([c[0] for c in cases], np.int32)
    cy = np.array([c[1] for c in cases], np.int32)
    X = np.array([c[2] for c in cases], np.int32)
    Y = np.array([c[3] for c in cases], np.int32)
    s, t = np.zeros(n), np.zeros(n)
    lib.quad_st(cx.ctypes.data_as(ctypes.c_void_p), cy.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(n), X.ctypes.data_as(ctypes.c_void_p),
                Y.ctypes.data_as(ctypes.c_void_p), s.ctypes.data_as(ctypes.c_void_p), t.ctypes.data_as(ctypes.c_void_p))
    clamped = centred = 0
    for i, (qx, qy, x, y) in enumerate(cases):
        want = rule_st(qx, qy, x, y)
        assert (s[i], t[i]) == want and 0 <= s[i] <= 1 and 0 <= t[i] <= 1, (qx, qy, x, y, (s[i], t[i]), want)
        centred += want == (0.5, 0.5)
        clamped += want[0] in (0.0, 1.0) or want[1] in (0.0, 1.0)
    assert centred > 100 and clamped > 1000
    # the corners themselves: tl (0, 0), tr (1, 0), br (1, 1), bl (0, 1) of a square, measured at the corners' centres
    sq = [(10, 10), (14, 10), (14, 14), (10, 14)]
    assert rule_st([p[0] for p in sq], [p[1] for p in sq], 10, 10) == (0.0, 0.0)
    assert rule_st([p[0] for p in sq], [p[1] for p in sq], 15, 15) == (1.0, 1.0)


def geom_of(host, w, h, ps):
    p = params_of(host, w, h, ps)
    g = FwdGeom()
    g.width, g.height, g.ps, g.numplates = w, h, ps, host.numplates
    g.rubix_block, g.rubix_pad, g.rubix_unit_px = p.rubix_block, p.rubix_pad, p.rubix_unit_px
    for i in range(6):
        g.plates[i] = p.plates[i]
    return g


def test_the_quad_ray_follows_the_rule(host, lib):
    host.command("f_globe tetra")
    g = geom_of(host, 8, 8, 16)
    plates = host.plates()
    cases = synthetic_quads()[::7]
    n = len(cases)
    cx = np.array([c[0] for c in cases], np.int32)
    cy = np.array([c[1] for c in cases], np.int32)
    X = np.array([c[2] for c in cases], np.int32)
    Y = np.array([c[3] for c in cases], np.int32)
    for plate, ps, tx, ty in [(0, 16, 0, 0), (1, 16, 15, 15), (2, 5, 3, 1), (3, 2048, 1023, 7)]:
        rays = np.zeros((n, 3), np.float32)
        lib.quad_ray(ctypes.byref(g), plate, ps, tx, ty, cx.ctypes.data_as(ctypes.c_void_p), cy.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(n),
                     X.ctypes.data_as(ctypes.c_void_p), Y.ctypes.data_as(ctypes.c_void_p), rays.ctypes.data_as(ctypes.c_void_p))
        for i, (qx, qy, x, y) in enumerate(cases):
            want = rule_ray(plates[plate], ps, tx, ty, *rule_st(qx, qy, x, y))
            assert np.array_equal(rays[i].view(np.uint32), want.view(np.uint32)), (plate, qx, qy, x, y, rays[i], want)


# ---- the device pipeline on the CPU ----------------------------------------------------------------------------------

def plate_ray(plates, plate, u, v):
    """FisheyeHost::plate_uv_to_ray in float32"""
    return rule_ray(plates[plate], 1, 0, 0, u + 0.5, v + 0.5)


def emulated_rays(host, fwd_unit, w, h, ps, order_seed):
    """the field the device path writes for the current lens and globe, emulated: (rays [h, w, 3], grid points settled)"""
    p = params_of(host, w, h, ps)
    n1, P = ps + 1, host.numplates
    npts = P * n1 * n1
    grid = np.zeros((npts, 2), np.int32)
    status = np.zeros(npts, np.uint8)
    undecided = np.zeros(npts, np.uint32)
    counters = np.zeros(16, np.uint32)
    fwd_unit.run_lt_forward_points(ctypes.byref(p), grid.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p),
                                   undecided.ctypes.data_as(ctypes.c_void_p), counters.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint(npts))
    plates = host.plates()
    und = undecided[: int(counters[0])]
    patches = (ForwardPatch * max(1, len(und)))()
    for k, pt in enumerate(und.tolist()):
        i, j, plate = pt % n1, pt // n1 % n1, pt // n1 // n1
        ray = plate_ray(plates, plate, (i - 0.5) / ps, (j - 0.5) / ps)
        st, (x, y) = host.lens_forward(float(ray[0]), float(ray[1]), float(ray[2]))
        patches[k].point, patches[k].status = pt, st
        if st == 1:
            patches[k].lx, patches[k].ly = x86_int(x / host.scale + w // 2), x86_int(-y / host.scale + h // 2)
    any_nil = int(counters[1] > 0 or any(patches[k].status != 1 for k in range(len(und))))
    owner = None
    if host.globe_name == "fast":   # a globe_plate globe: the owner plane, from the interpreter
        owner = np.zeros(P * ps * ps, np.uint8)
        for plate in range(P):
            for py in range(ps):
                for px in range(ps):
                    r = plate_ray(plates, plate, px / ps, py / ps)
                    _, sel = host.globe_plate(float(r[0]), float(r[1]), float(r[2]))
                    owner[(plate * ps + py) * ps + px] = sel == plate
    order = np.random.default_rng(order_seed).permutation(P * ps * ps).astype(np.uint32)
    rays = np.full((h, w, 3), np.float32(12345.0))
    lib = emulated_rays.lib
    lib.run_rays(ctypes.byref(geom_of(host, w, h, ps)), grid.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p), patches,
                 ctypes.c_uint(len(und)), any_nil, None if owner is None else owner.ctypes.data_as(ctypes.c_void_p),
                 order.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint(len(order)), rays.ctypes.data_as(ctypes.c_void_p))
    return rays, len(und)


def assert_same_bytes(got, want, what=""):
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32, what
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (what, len(bad), [(tuple(i), got[tuple(i)], want[tuple(i)]) for i in bad[:4]])


@pytest.mark.parametrize("lens", FORWARD_ONLY + ["holes"])
def test_the_emulated_device_pipeline_equals_the_host_export(host, lib, tmp_path, lens):
    emulated_rays.lib = lib
    host.set_rubixgrid(*GRID)
    unit = None
    sizes = {"cube": (128, 80, 20), "fast": (97, 61, 14), "tetra": (1, 33, 9)}
    if lens in ("sinusoidal", "holes"):
        sizes["trism"] = (47, 1, 9)
    for seed, (globe, (w, h, ps)) in enumerate(sizes.items()):
        host.command(f"f_globe {globe}")
        if lens == "holes":
            host.load_lens("holes", HOLES)
        else:
            host.command(f"f_lens {lens}")
        want = host.raymap(w, h, forward=True, platesize=ps)
        assert host.build_info.startswith("ray export (forward), host"), host.build_info
        host.build_lensmap(w, h, ps, threads=1)   # the scale, for params_of
        if unit is None:   # lens_forward and the grid-point kernel, translated on cube: the same points on every globe
            unit = build_lib(host.lens_source(forward=True, with_kernel=True), RUN_FORWARD, str(tmp_path / lens))
        got, _ = emulated_rays(host, unit, w, h, ps, seed)
        assert_same_bytes(got, want, (lens, globe))
        idx, _ = host.lensmap()
        assert np.array_equal(np.any(want != 0, axis=2), idx >= 0), (lens, globe, "mapped exactly where the build maps")


# ---- what the rays are -------------------------------------------------------------------------------------------------

def plate_uv(plates, plate, rays):
    """(u, v) [n] of rays [n, 3] projected on plate (ray_to_plate_uv in float64)"""
    f, r, up = (np.asarray(plates[plate][k:k + 3], np.float64) for k in (0, 3, 6))
    d = 0.5 / math.tan(float(np.float32(plates[plate][9]) / np.float32(2)))
    rr = rays.astype(np.float64)
    z = rr @ f
    return (rr @ r) / z * d + 0.5, -(rr @ up) / z * d + 0.5


@pytest.mark.parametrize("globe", ["cube", "fast"])
def test_each_ray_lies_in_its_winning_texels_quad(host, globe):
    W, H, ps = 320, 180, 96
    host.command(f"f_globe {globe}")
    plates = host.plates()
    for lens in FORWARD_ONLY[::3]:
        host.command(f"f_lens {lens}")
        rays = host.raymap(W, H, forward=True, platesize=ps)
        host.build_lensmap(W, H, ps, threads=1)
        idx, _ = host.lensmap()
        mapped = idx >= 0
        assert np.array_equal(np.any(rays != 0, axis=2), mapped), lens
        i = idx[mapped].astype(np.int64)
        plate, rest = np.divmod(i, ps * ps)
        ty, tx = np.divmod(rest, ps)
        r = rays[mapped]
        assert np.allclose(np.linalg.norm(r.astype(np.float64), axis=1), 1, atol=1e-6), lens
        for P in np.unique(plate):
            m = plate == P
            u, v = plate_uv(plates, int(P), r[m])
            eps = 1e-5
            assert (u >= (tx[m] - 0.5) / ps - eps).all() and (u <= (tx[m] + 0.5) / ps + eps).all(), (lens, int(P))
            assert (v >= (ty[m] - 0.5) / ps - eps).all() and (v <= (ty[m] + 0.5) / ps + eps).all(), (lens, int(P))


def round_trip(host, rays, W, H):
    """for every mapped pixel: the distance in pixels (max of |dx|, |dy|) from the pixel to where lens_forward puts its
    ray, measured at the pixel's continuous position"""
    ys, xs = np.nonzero(np.any(rays != 0, axis=2))
    d = np.zeros(len(ys))
    for k, (y, x) in enumerate(zip(ys.tolist(), xs.tolist())):
        st, (fx, fy) = host.lens_forward(*(float(c) for c in rays[y, x]))
        assert st == 1, (x, y)
        d[k] = max(abs(fx / host.scale + W // 2 - x), abs(-fy / host.scale + H // 2 - y))
    return d


# measured on cube at 640x360, platesize 360, over all ten lenses and three zooms (DESIGN §3h): median 0.57-0.77 px,
# 99th percentile up to 2.10 px, maximum up to 17.0 px (pixels beside the seams of the whole-sphere maps)
ROUND_TRIP_MEDIAN = 0.8
ROUND_TRIP_P99 = 2.25
ROUND_TRIP_MAX = 18.0


@pytest.mark.parametrize("zoom", ["f_fov 180", "f_cover", "f_contain"])
def test_round_trip_through_lens_forward(host, zoom):
    W, H = 640, 360
    host.command("f_globe cube")
    measured = {}
    for lens in FORWARD_ONLY:
        host.command(f"f_lens {lens}")
        host.command(zoom)
        try:
            rays = host.raymap(W, H, forward=True)
        except Exception as e:  # noqa: BLE001 — a zoom this lens cannot do (polyconic has no lens_width for f_cover)
            assert "zoom could not be computed" in str(e), (lens, str(e))
            continue
        host.build_lensmap(W, H, 0, threads=1)   # the same build: its scale for the round trip, its map for mapped-ness
        idx, _ = host.lensmap()
        assert np.array_equal(np.any(rays != 0, axis=2), idx >= 0), (lens, zoom)
        d = round_trip(host, rays, W, H)
        measured[lens] = (float(np.median(d)), float(np.quantile(d, 0.99)), float(d.max()))
        assert np.median(d) <= ROUND_TRIP_MEDIAN and np.quantile(d, 0.99) <= ROUND_TRIP_P99 and d.max() <= ROUND_TRIP_MAX, (lens, zoom, measured[lens])
    assert len(measured) >= 9, measured


# the angle between the forward and the inverse export of a pixel, in pixel pitches (the larger angle to its right or lower
# neighbour's inverse ray), measured at 640x360 on cube (DESIGN §3h): median 0.63-0.69, 99th percentile 1.21-1.49,
# maximum 1.48-5.11 (hammer, beside its rim)
ANGLE_MEDIAN = 0.75
ANGLE_P99 = 1.75
ANGLE_MAX = 6.0


@pytest.mark.parametrize("lens,zoom", [("equirect", "f_contain"), ("hammer", "f_contain"), ("mercator", "f_fov 180"), ("panini", "f_fov 180")])
def test_lenses_with_both_functions_agree_with_their_inverse_export(host, lens, zoom):
    W, H = 640, 360
    host.command("f_globe cube")
    host.command(f"f_lens {lens}")
    host.command(zoom)
    fwd = host.raymap(W, H, forward=True).astype(np.float64)
    with np.errstate(all="ignore"):
        inv = host.raymap(W, H).astype(np.float64)
        inv /= np.linalg.norm(inv, axis=2, keepdims=True)   # (nil pixels become NaN and drop out)

    def angle(a, b):
        return np.arccos(np.clip(np.sum(a * b, axis=-1), -1, 1))

    pitch = np.full((H, W), np.nan)
    pitch[:, :-1] = angle(inv[:, :-1], inv[:, 1:])
    pitch[:-1] = np.fmax(pitch[:-1], angle(inv[:-1], inv[1:]))
    both = np.any(fwd != 0, axis=2) & np.all(np.isfinite(inv), axis=2) & np.isfinite(pitch) & (pitch > 0)
    assert both.mean() > 0.3, (lens, both.mean())
    ratio = angle(fwd[both], inv[both]) / pitch[both]
    q = (float(np.median(ratio)), float(np.quantile(ratio, 0.99)), float(ratio.max()))
    assert q[0] <= ANGLE_MEDIAN and q[1] <= ANGLE_P99 and q[2] <= ANGLE_MAX, (lens, zoom, q)


# ---- refusals and state ----------------------------------------------------------------------------------------------

def test_refusals(bb, host):
    lib = bb.load_library()
    buf = np.zeros(3 * 64 * 64 + 1, np.float32)
    ptr = buf.ctypes.data
    assert lib.blinky_get_raymap_forward(host._ctx, 8, 8, 0, ptr) == bb.E_STATE, "no lens"
    host.command("f_lens sinusoidal")
    assert lib.blinky_get_raymap_forward(host._ctx, 8, 8, 0, ptr) == bb.E_STATE, "no globe"
    assert "no valid globe" in lib.blinky_last_error(host._ctx).decode()
    host.command("f_globe cube")
    host.build_lensmap(32, 24, 16, threads=1)
    before, info = state(host), host.build_info
    for what, w, h, ps, p in [("NULL rays", 8, 8, 0, None), ("misaligned", 8, 8, 0, ptr + 2), ("width 0", 0, 8, 0, ptr), ("height < 0", 8, -1, 0, ptr),
                              ("platesize over the limit", 8, 8, 6689, ptr)]:
        assert lib.blinky_get_raymap_forward(host._ctx, w, h, ps, p) == bb.E_INVALID, what
        assert_same_state(before, state(host))
        assert host.build_info == info
    assert lib.blinky_get_raymap_forward(host._ctx, 8, 8, 6688, ptr) == bb.OK, "6 * 6688^2 < 2^28"
    # the default platesize min(W, H) at 4K with k = 4 is beyond the limit: such an export names its platesize
    assert lib.blinky_get_raymap_forward(host._ctx, 4 * 3840, 4 * 2160, 0, ptr) == bb.E_INVALID
    assert lib.blinky_get_raymap_forward_device(host._ctx, 8, 8, 0, ptr, None) == bb.E_NODEVICE
    # the inverse export keeps refusing forward lenses
    with pytest.raises(bb.BlinkyError, match="no per-pixel ray") as e:
        host.raymap(8, 8)
    assert e.value.code == bb.E_STATE
    # a lens without lens_forward
    host.load_lens("inv", "lens_width = 2\nfunction lens_inverse(x, y) return x, y, 1 end")
    assert lib.blinky_get_raymap_forward(host._ctx, 8, 8, 0, ptr) == bb.E_STATE
    assert "lens_forward" in lib.blinky_last_error(host._ctx).decode()
    # a zoom the lens cannot do
    host.command("f_lens polyconic")
    host.command("f_cover")
    host.clear_log()
    assert lib.blinky_get_raymap_forward(host._ctx, 8, 8, 0, ptr) == bb.E_ZOOM
    assert host.log
    # a raising lens_forward
    host.load_lens("bad", "map = 'lens_forward'\nmax_fov = 360\nmax_vfov = 180\nlens_width = 2\n"
                          "function lens_forward(x, y, z) if x > 0.5 then error('boom') end return x, y end")
    host.command("f_contain")
    host.clear_log()
    assert lib.blinky_get_raymap_forward(host._ctx, 64, 8, 0, ptr) == bb.E_SCRIPT
    assert "boom" in host.log, host.log
    assert_same_state(before, state(host))


def test_an_export_changes_nothing(host):
    W, H, ps = 96, 64, 32
    host.command("f_globe cube")
    host.command("f_lens winkel1")
    host.build_lensmap(W, H, ps, threads=1)
    before, scale, display = state(host), host.scale, host.display()
    host.clear_log()
    rays = host.raymap(200, 100, forward=True, platesize=48)
    assert np.any(rays != 0)
    assert_same_state(before, state(host))
    assert host.scale == scale and host.display() == display and (host.width, host.height, host.platesize) == (W, H, ps)
    assert not host.needs_rebuild(W, H, ps)
    assert host.log == "", "no '> maxdiff' lines or anything else"
    host.command("f_lens gins8")
    host.command("f_globe trism")
    assert host.needs_rebuild(W, H, ps)
    host.raymap(W, H, forward=True)
    assert host.needs_rebuild(W, H, ps), "pending changes stay pending"
    assert_same_state(before, state(host))


def test_the_new_symbols_are_declared_and_exported(bb):
    from test_capi import declared_symbols

    lib = ctypes.CDLL(bb.LIB_PATH)
    for name in ("blinky_get_raymap_forward", "blinky_get_raymap_forward_device"):
        assert name in declared_symbols() and name in bb.EXPORTED_SYMBOLS and hasattr(lib, name), name
