"""Globes that pick their plates with a `globe_plate(x, y, z)` script (the `fast` globe) on the device
lensmap builder: the translator turns globe_plate into `lt_globe_plate` in the lens's translation unit,
the inverse kernel lets it pick the plate, and the forward builder gets an owner kernel.

CPU suite, like test_transpile.py / test_device_emulation.py: the translated source is compiled with g++
(host libm, or every libm result moved by pseudo-random ulps as another libm would) and must give the
interpreter's plate for every ray it does not flag, and the emulated device builds must merge into the
interpreter's lensmap."""
import ctypes
import math

import numpy as np
import pytest

from test_device_emulation import GRID, RUN_FORWARD, RUN_INVERSE, ForwardPatch, FwdGeom, LtParams, build_lib, x86_int
from test_transpile import FORWARD_ONLY, TRANSLATABLE, perturbed

WRAP_GP = r"""
extern "C" int gp_eval(double x, double y, double z, int *plate, unsigned *flag) {
    Ctx c; c.flag = 0; c.steps = 0; c.plates = 0; c.numplates = 0;
    lt_init_mut(c);
    const int ok = lt_globe_plate(c, x, y, z, plate) ? 1 : 0;
    *flag = c.flag;
    return ok;
}
"""

RUN_OWNER = r"""
extern "C" void run_lt_forward_owner(const LtParams *P, unsigned char *owner, unsigned *undecided, unsigned *counter, unsigned cap) {
    blockDim.x = 128; blockDim.y = blockDim.z = 1;
    const unsigned ps = P->platesize;
    for (unsigned bz = 0; bz < (unsigned)P->numplates; ++bz)
        for (unsigned by = 0; by < ps; ++by)
            for (unsigned bx = 0; bx * 128 < ps; ++bx)
                for (unsigned t = 0; t < 128; ++t) {
                    blockIdx.x = bx; blockIdx.y = by; blockIdx.z = bz; threadIdx.x = t;
                    lt_forward_owner(*P, owner, undecided, counter, cap);
                }
}
"""

# ----------------------------------------------------------------------------- custom globes

TWO_PLATES = """
plates = {
  { {0,0,1}, {0,1,0}, 120 },
  { {0,0,-1}, {0,1,0}, 120 },
}
"""

CUSTOM_GLOBES = {
    # lua_tointeger truncates: 1.5 -> 1, -0.5 -> 0, 0.9999999 -> 0
    "fractions": TWO_PLATES + """
function globe_plate(x, y, z)
  if x > 0.2 then return 1.5 end
  if x < -0.2 then return -0.5 end
  return 0.9999999
end""",
    # NaN and out-of-int-range values convert differently on x86 and CUDA: always the interpreter's
    "nan_huge": TWO_PLATES + """
function globe_plate(x, y, z)
  if x > 0.3 then return 0/0 end
  if x < -0.3 then return 1e12 end
  if y > 0.3 then return -1e12 end
  return 1
end""",
    # plates 2..5 of a 2-plate globe: whatever the previous globe (cube) left in those slots
    "stale": TWO_PLATES + """
function globe_plate(x, y, z)
  if z > 0.7 then return 0 end
  if z < -0.7 then return 1 end
  if x > 0.3 then return 2 end
  if x < -0.3 then return 3 end
  if y > 0 then return 4 end
  return 5
end""",
    # a script-level variable written by globe_plate (a per-pixel slot on the device)
    "mutable": TWO_PLATES + """
last_z = 0
function globe_plate(x, y, z)
  last_z = z * 2
  if last_z > 0.25 then return 0 end
  return 1
end""",
    # libm inside globe_plate: the decision near lon = +-1.2 carries an error bound
    "latlon": TWO_PLATES + """
function globe_plate(x, y, z)
  local lat, lon = ray_to_latlon(x, y, z)
  if abs(lon) < 1.2 and lat < 0.9 then return 7, 0 end
  return 7, 1   -- the last value counts
end""",
    # a global helper that both globe_plate and the lens (HELPER_LENS) call
    "helper": TWO_PLATES + """
function blend(a, b)
  return a * 0.75 + b * sin(a)
end
function globe_plate(x, y, z)
  if blend(z, x) > 0 then return 0 end
  return 1
end""",
}

HELPER_LENS = """
onload = "f_contain"
lens_height = pi
lens_width = 2*pi
max_vfov = 180
max_fov = 360
function lens_inverse(x, y)
  if abs(y) > pi/2 or abs(x) > pi then return nil end
  return latlon_to_ray(y, blend(x, 0) * 1.3)
end
"""

REFUSED_GLOBES = [
    (TWO_PLATES + "function globe_plate(x, y, z) return x > 0 end", "booleans"),
    (TWO_PLATES + "function globe_plate(x, y, z) if x > 0 then return '1' end return 0 end", "string"),
    (TWO_PLATES + "function globe_plate(x, y, z) local f = function() return 1 end return f() end", "closures"),
]


def load_custom(host, name):
    """loads custom globe `name` (right after the cube globe for "stale") and its lens; returns the six
    plate slots the host holds: the new globe's plates, then what the earlier globe left"""
    host.command("f_globe cube")
    slots = np.zeros((6, 11), np.float32)
    slots[:6] = host.plates()
    host.load_globe(name, CUSTOM_GLOBES[name])
    pl = host.plates()
    slots[: len(pl)] = pl
    if name == "helper":
        host.load_lens("helper_lens", HELPER_LENS)
    else:
        host.command("f_lens equirect")
    return slots


# ----------------------------------------------------------------------------- helpers


def gp_lib(host, tmp_path, tag, scale=0):
    src = host.lens_source(cuda=False, globe_plate=True)
    if scale:
        src = perturbed(src, scale)
    lib = build_lib(src, WRAP_GP, str(tmp_path / f"gp_{tag}_{scale}"))
    lib.gp_eval.argtypes = [ctypes.c_double] * 3 + [ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint)]
    return lib


def fast_rays():
    """float32 rays: random unit rays, the axes, z <= 0, and rays on both sides of the small plate's edge |u| = size/2
    (fast.lua: |x/z| = tan(pi/4) in the big plate's frame)"""
    rng = np.random.default_rng(17)
    r = rng.normal(size=(1500, 3))
    r /= np.linalg.norm(r, axis=1, keepdims=True)
    rays = [r.astype(np.float32)]
    axes = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [0, 0, 0]], np.float32)
    rays.append(axes)
    back = rng.normal(size=(200, 3))
    back[:, 2] = -np.abs(back[:, 2])
    back[:20, 2] = 0.0
    back[20:40, 2] = -0.0
    rays.append(back.astype(np.float32))
    edge = []
    for _ in range(70):
        z = np.float32(rng.uniform(0.1, 1.0))
        w = np.float32(z * rng.uniform(-0.9, 0.9))
        for k in range(-3, 4):
            e = np.float32(z)
            for _ in range(abs(k)):
                e = np.nextafter(e, np.float32(np.inf if k > 0 else 0), dtype=np.float32)
            edge.append((e, w, z))   # |u| edge
            edge.append((-e, w, z))
            edge.append((w, e, z))   # |v| edge
    rays.append(np.array(edge, np.float32))
    return np.vstack(rays)


def params6(host, w, h, ps, slots):
    """LtParams of FisheyeHost::device_params: all six plate slots, uv_dist = 0.5 / tan(fov/2) (inf for fov 0)"""
    p = LtParams()
    p.width, p.height, p.platesize, p.numplates = w, h, ps, host.numplates
    p.scale = host.scale
    numcells, cell, pad = GRID
    p.rubix_block = pad + cell
    p.rubix_pad = pad
    p.rubix_unit_px = float(ps) / (numcells * p.rubix_block + pad)
    for i, row in enumerate(slots):
        for k in range(3):
            p.plates[i].forward[k], p.plates[i].right[k], p.plates[i].up[k] = row[k], row[3 + k], row[6 + k]
        p.plates[i].dist = row[10]
        t = math.tan(float(np.float32(row[9]) / np.float32(2)))  # float halving, double tan (fisheye.c:2060)
        p.uv_dist[i] = 0.5 / t if t != 0 else math.inf
    return p


def emulated_inverse(host, tmp_path, tag, w, h, ps, slots, scale):
    """(candidates' idx, tint, risk) of the NVRTC text run behind the CPU shim"""
    src = host.lens_source(with_kernel=True)
    assert "#define LT_HAS_GLOBE_PLATE 1" in src and "lt_globe_plate(c, (double)ray[0]" in src
    if scale:
        src = perturbed(src, scale)
    lib = build_lib(src, RUN_INVERSE, str(tmp_path / f"inv_{tag}_{scale}"))
    p = params6(host, w, h, ps, slots)
    cand = np.zeros(w * h, np.uint32)
    lib.run_lt_build(ctypes.byref(p), cand.ctypes.data_as(ctypes.c_void_p))
    cand = cand.reshape(h, w)
    risk = (cand & 0x20000000) != 0
    valid = (cand & 0x80000000) != 0
    ongrid = (cand & 0x40000000) != 0
    c_idx = np.where(valid, (cand & 0x0FFFFFFF).astype(np.int64), -1)
    c_tint = np.where(valid & ~ongrid, c_idx // (ps * ps), 255)
    return c_idx, c_tint, risk


def texel_rays(slots, numplates, ps):
    """plate_uv_to_ray(plate, px/ps, py/ps) in float32, exactly as build_forward / fwd_raster_texel make it:
    [numplates, ps(py), ps(px), 3]"""
    out = np.zeros((numplates, ps, ps, 3), np.float32)
    u = (np.arange(ps, dtype=np.float64) / ps - 0.5).astype(np.float32)
    v = (-(np.arange(ps, dtype=np.float64) / ps - 0.5)).astype(np.float32)
    U, V = np.meshgrid(u, v)
    for p in range(numplates):
        f, r, up = (slots[p][k:k + 3].astype(np.float32) for k in (0, 3, 6))
        dist = np.float32(slots[p][10])
        ray = [np.float32(0) + dist * f[k] + np.zeros_like(U) for k in range(3)]
        ray = [ray[k] + U * r[k] for k in range(3)]
        ray = [ray[k] + V * up[k] for k in range(3)]
        ln = (ray[0] * ray[0] + ray[1] * ray[1]) + ray[2] * ray[2]
        ln = np.sqrt(ln.astype(np.float64)).astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = np.where(ln != 0, np.float32(1) / ln, np.float32(1))
        for k in range(3):
            out[p, :, :, k] = np.where(ln != 0, ray[k] * inv, ray[k])
    return out


def host_owner(host, rays, numplates, ps):
    own = np.zeros((numplates, ps, ps), np.uint8)
    for p in range(numplates):
        for py in range(ps):
            for px in range(ps):
                x, y, z = rays[p, py, px]
                st, plate = host.globe_plate(float(x), float(y), float(z))
                own[p, py, px] = st == 1 and plate == p
    return own


# ----------------------------------------------------------------------------- 1, 2: the translated globe_plate


def test_fast_globe_plate_translation_is_exact(host, tmp_path):
    host.command("f_globe fast")
    host.command("f_lens panini")
    lib = gp_lib(host, tmp_path, "fast")
    rays = fast_rays()
    assert len(rays) >= 2000
    plate, flag = ctypes.c_int(), ctypes.c_uint()
    flagged = 0
    seen = set()
    for x, y, z in rays.astype(np.float64):
        st, want = host.globe_plate(x, y, z)
        ok = lib.gp_eval(x, y, z, ctypes.byref(plate), ctypes.byref(flag))
        assert (st, want) == (ok, plate.value), (x, y, z)
        flagged += bool(flag.value)
        seen.add(want)
    assert seen == {-1, 0, 1}
    assert flagged <= 0.1 * len(rays), flagged


@pytest.mark.parametrize("scale", [1, 1 << 20])
def test_fast_globe_plate_bounds_are_sound(host, tmp_path, scale):
    host.command("f_globe fast")
    host.command("f_lens panini")
    lib = gp_lib(host, tmp_path, "fast", scale)
    rays = fast_rays()
    plate, flag = ctypes.c_int(), ctypes.c_uint()
    decided = 0
    for x, y, z in rays.astype(np.float64):
        ok = lib.gp_eval(x, y, z, ctypes.byref(plate), ctypes.byref(flag))
        if flag.value:
            continue
        decided += 1
        assert host.globe_plate(x, y, z) == (ok, plate.value), (scale, x, y, z)
    assert decided >= 0.8 * len(rays), (scale, decided)


def test_globe_plate_source_flavours(bb, host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    with pytest.raises(bb.BlinkyError, match="no globe_plate"):
        host.lens_source(globe_plate=True)
    assert host.globe_plate(0, 0, 1) == (-2, -1)
    assert "lt_globe_plate" not in host.lens_source(with_kernel=True)
    host.command("f_globe fast")
    alone = host.lens_source(cuda=True, globe_plate=True)
    assert "__device__" in alone and "lt_globe_plate" in alone and "lt_entry" not in alone
    # without the kernel: the lens alone, as before; with it: one unit with globe_plate
    assert "lt_globe_plate" not in host.lens_source()
    src = host.lens_source(with_kernel=True)
    assert src.count("#define LT_HAS_GLOBE_PLATE 1") == 1 and "lt_entry" in src
    fwd = host.lens_source(cuda=True, forward=True, with_kernel=True)
    assert "lt_forward_owner" in fwd


def test_globe_plate_compiles_for_sm90a(bb, host):
    host.command("f_globe fast")
    for lens, forward in [("panini", False), ("quincuncial", False), ("sinusoidal", True)]:
        host.command(f"f_lens {lens}")
        try:
            size = host.compile_lens(forward=forward)
        except bb.BlinkyError as e:
            if "NVRTC not found" in str(e):
                pytest.skip(str(e))
            raise
        assert size > 1000


# ----------------------------------------------------------------------------- 3: emulated inverse builds on `fast`


@pytest.mark.parametrize("scale", [0, 1, 1 << 20])
@pytest.mark.parametrize("lens", TRANSLATABLE)
def test_emulated_inverse_build_on_fast_equals_interpreter(host, tmp_path, lens, scale):
    w, h, ps = 96, 64, 48
    host.set_rubixgrid(*GRID)
    host.command("f_globe fast")
    host.command(f"f_lens {lens}")
    host.build_lensmap(w, h, ps, threads=1)
    idx, tint = host.lensmap()
    slots = np.zeros((6, 11), np.float32)  # a fresh context: slots 2..5 were never filled
    slots[:2] = host.plates()
    c_idx, c_tint, risk = emulated_inverse(host, tmp_path, lens, w, h, ps, slots, scale)
    got_idx = np.where(risk, idx, c_idx)
    got_tint = np.where(risk, tint, c_tint)
    assert np.array_equal(got_idx, idx), (lens, scale, int((got_idx != idx).sum()))
    assert np.array_equal(got_tint, tint), (lens, scale)
    if scale == 0:
        assert np.array_equal(c_idx, idx) and np.array_equal(c_tint, tint), lens
    assert risk.mean() < (0.25 if scale <= 1 else 0.98), (lens, scale, float(risk.mean()))


# ----------------------------------------------------------------------------- 4: custom globes


@pytest.mark.parametrize("scale", [0, 1 << 20])
@pytest.mark.parametrize("name", sorted(CUSTOM_GLOBES))
def test_emulated_build_with_custom_globe_plate_equals_interpreter(host, tmp_path, name, scale):
    w, h, ps = 96, 64, 40
    host.set_rubixgrid(*GRID)
    slots = load_custom(host, name)
    host.build_lensmap(w, h, ps, threads=1)
    idx, tint = host.lensmap()
    assert (idx >= 0).sum() > 0.1 * w * h, name
    c_idx, c_tint, risk = emulated_inverse(host, tmp_path, name, w, h, ps, slots, scale)
    got_idx = np.where(risk, idx, c_idx)
    got_tint = np.where(risk, tint, c_tint)
    assert np.array_equal(got_idx, idx), (name, scale, int((got_idx != idx).sum()))
    assert np.array_equal(got_tint, tint), (name, scale)
    if name == "stale":
        assert (idx >= 2 * ps * ps).any()  # the map really reads the slots behind the globe's two plates
    if name == "nan_huge":
        assert risk.any()


def test_custom_globe_plate_translation_details(host):
    load_custom(host, "helper")
    src = host.lens_source(with_kernel=True)
    assert src.count("_blend(Ctx &c") == 1  # one function table: the shared helper is emitted once
    load_custom(host, "mutable")
    src = host.lens_source(with_kernel=True)
    assert "c.mg[0] = " in src
    load_custom(host, "latlon")
    assert "lt_plate_int(c, r[1])" in host.lens_source(globe_plate=True)  # the last value returned counts


@pytest.mark.parametrize("src, why", REFUSED_GLOBES)
def test_untranslatable_globe_plate_says_why(bb, host, src, why):
    host.load_globe("t", src)
    host.command("f_lens equirect")
    with pytest.raises(bb.BlinkyError, match=why):
        host.lens_source(globe_plate=True)
    with pytest.raises(bb.BlinkyError, match="globe_plate: .*" + why):
        host.lens_source(with_kernel=True)
    host.lens_source()  # the lens alone still translates


# ----------------------------------------------------------------------------- 5: forward owner pass on `fast`

FWD_OWNER_HARNESS = r"""
#include <vector>
#include <cstring>
#include "forward_raster.h"
using namespace blinky;
extern "C" void fwd_run_owner(const FwdGeom *g, FwdPoint *grid, unsigned char *status, const ForwardPatch *patches, unsigned npatch,
                              int any_nil, unsigned char *owner, const uint32_t *owner_patches, unsigned nowner, int32_t *idx,
                              uint8_t *tint, int *display, FwdMessage *messages, unsigned *nmsg) {
    for (unsigned k = 0; k < npatch; ++k) fwd_apply_patch(grid, status, patches[k]);
    for (unsigned k = 0; k < nowner; ++k) fwd_apply_owner_patch(owner, owner_patches[k]);
    if (any_nil)
        for (int t = 2 * (g->ps + 1) - 1; t >= 0; --t) fwd_stale_chain(grid, status, g->ps, g->numplates, t);
    const size_t npix = (size_t)g->width * g->height;
    std::vector<unsigned> keys(2 * npix, 0u);
    unsigned counters[16];
    memset(counters, 0, sizeof counters);
    FwdOut o{keys.data(), keys.data() + npix, counters, messages};
    for (int plate = g->numplates - 1; plate >= 0; --plate)
        for (int py = 0; py < g->ps; ++py)
            for (int px = g->ps - 1; px >= 0; --px) fwd_raster_texel(*g, grid, o, plate, py, px, owner);
    for (size_t at = 0; at < npix; ++at) fwd_resolve_pixel(keys.data(), keys.data() + npix, idx, tint, at, g->ps);
    for (int i = 0; i < 6; ++i) display[i] = counters[3 + i] ? 1 : 0;
    *nmsg = counters[2];
}
"""


@pytest.fixture(scope="module")
def fwd_owner_lib(tmp_path_factory):
    import os
    import subprocess

    d = tmp_path_factory.mktemp("fwd_owner")
    src = d / "fwd_owner.cpp"
    src.write_text(FWD_OWNER_HARNESS)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(root, "blinky_b200", "csrc"),
                        "-o", str(d / "fwd_owner.so"), str(src)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:3000]
    return ctypes.CDLL(str(d / "fwd_owner.so"))


def grid_point_ray(plates, ps, pt):
    n1 = ps + 1
    i, j, plate = pt % n1, pt // n1 % n1, pt // n1 // n1
    f, r, u = (plates[plate][a:a + 3].astype(np.float32) for a in (0, 3, 6))
    uu = np.float32((i - 0.5) / ps - 0.5)
    vv = np.float32(-((j - 0.5) / ps - 0.5))
    ray = np.float32(plates[plate][10]) * f
    ray = ray + uu * r
    ray = ray + vv * u
    ln = np.float32(math.sqrt(float(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2])))
    if ln:
        ray = ray * (np.float32(1) / ln)
    return ray


@pytest.mark.parametrize("scale", [0, 1 << 20])
@pytest.mark.parametrize("lens", FORWARD_ONLY)
def test_emulated_forward_owner_pass_on_fast(host, fwd_owner_lib, tmp_path, lens, scale):
    """owner kernel (NVRTC text behind the shim) + the host's answers for its flagged texels == the host's
    per-texel ownership; then the whole forward build with that owner plane == the serial host builder"""
    w, h, ps = 128, 80, 24
    host.set_rubixgrid(*GRID)
    host.command("f_globe fast")
    host.command(f"f_lens {lens}")
    host.clear_log()
    host.build_lensmap(w, h, ps, threads=1)
    want_idx, want_tint = host.lensmap()
    want_disp, want_log = host.display(), host.log
    P = host.numplates
    slots = np.zeros((6, 11), np.float32)
    slots[:P] = host.plates()

    src = host.lens_source(forward=True, with_kernel=True)
    if scale:
        src = perturbed(src, scale)
    lib = build_lib(src, RUN_FORWARD + RUN_OWNER, str(tmp_path / f"{lens}_{scale}"))
    p = params6(host, w, h, ps, slots)
    ntex = P * ps * ps
    owner = np.zeros(ntex, np.uint8)
    und_t = np.zeros(ntex, np.uint32)
    cnt = np.zeros(1, np.uint32)
    lib.run_lt_forward_owner(ctypes.byref(p), owner.ctypes.data_as(ctypes.c_void_p), und_t.ctypes.data_as(ctypes.c_void_p),
                             cnt.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint(ntex))
    assert int(cnt[0]) == int(((owner & 2) != 0).sum())
    if scale == 0:
        assert int(cnt[0]) <= 0.05 * ntex
    rays = texel_rays(slots, P, ps)
    want_owner = host_owner(host, rays, P, ps).reshape(-1)
    # the host settles the flagged texels (FisheyeHost::build_forward_device)
    und_t = und_t[: int(cnt[0])]
    owner_patches = np.array([t | (0x80000000 if want_owner[t] else 0) for t in und_t.tolist()], np.uint32)
    patched = owner.copy()
    patched[und_t] = want_owner[und_t]
    assert np.array_equal(patched & 1, want_owner), (lens, scale, int(((patched & 1) != want_owner).sum()))

    # the rest of the forward pipeline with this owner plane
    n1 = ps + 1
    npts = P * n1 * n1
    grid = np.zeros((npts, 2), np.int32)
    status = np.zeros(npts, np.uint8)
    undecided = np.zeros(npts, np.uint32)
    counters = np.zeros(16, np.uint32)
    lib.run_lt_forward_points(ctypes.byref(p), grid.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p),
                              undecided.ctypes.data_as(ctypes.c_void_p), counters.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint(npts))
    und = undecided[: int(counters[0])]
    patches = (ForwardPatch * max(1, len(und)))()
    for k, pt in enumerate(und.tolist()):
        ray = grid_point_ray(slots, ps, pt)
        st, (x, y) = host.lens_forward(float(ray[0]), float(ray[1]), float(ray[2]))
        patches[k].point, patches[k].status = pt, st
        if st == 1:
            patches[k].lx, patches[k].ly = x86_int(x / host.scale + w // 2), x86_int(-y / host.scale + h // 2)
    any_nil = int(counters[1] > 0 or any(patches[k].status != 1 for k in range(len(und))))
    g = FwdGeom()
    g.width, g.height, g.ps, g.numplates = w, h, ps, P
    g.rubix_block, g.rubix_pad, g.rubix_unit_px = p.rubix_block, p.rubix_pad, p.rubix_unit_px
    for i in range(6):
        g.plates[i] = p.plates[i]
    idx = np.zeros(w * h, np.int32)
    tint = np.zeros(w * h, np.uint8)
    disp = (ctypes.c_int * 6)()
    msgs = np.zeros((4096, 2), np.uint32)
    nmsg = ctypes.c_uint()
    op = owner_patches if len(owner_patches) else np.zeros(1, np.uint32)
    fwd_owner_lib.fwd_run_owner(ctypes.byref(g), grid.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p), patches,
                                ctypes.c_uint(len(und)), any_nil, owner.ctypes.data_as(ctypes.c_void_p), op.ctypes.data_as(ctypes.c_void_p),
                                ctypes.c_uint(len(owner_patches)), idx.ctypes.data_as(ctypes.c_void_p), tint.ctypes.data_as(ctypes.c_void_p),
                                disp, msgs.ctypes.data_as(ctypes.c_void_p), ctypes.byref(nmsg))
    assert np.array_equal(idx.reshape(h, w), want_idx), (lens, scale, int((idx.reshape(h, w) != want_idx).sum()))
    assert np.array_equal(tint.reshape(h, w), want_tint), (lens, scale)
    assert list(disp)[:P] == want_disp[:P], lens
    got_log = "".join(f"{int(v)} > maxdiff\n" for _, v in sorted(map(tuple, msgs[: nmsg.value].tolist())))
    assert got_log == "".join(l + "\n" for l in want_log.splitlines() if l.endswith("> maxdiff")), lens
