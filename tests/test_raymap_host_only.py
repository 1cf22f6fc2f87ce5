"""Ray maps (blinky_set_raymap) on host-only contexts: a field of view rays, mapped through the current globe, gives
the lensmap a build gives for a lens that returns those rays.  Every inverse lens on every globe in the golden order
(so the stale plate slots are the golden builds'), against the build of the same context and the compiled
reference's fixtures; adversarial rays against the reference rule written out in numpy; the ray-map kernel's text
behind the CPU shim of test_device_emulation.py; refusals and state.  The GPU path is tests/test_gpu_raymap.py."""
import ctypes
import json
import math
import os

import numpy as np
import pytest

from test_device_emulation import GRID, build_lib
from test_globe_plate_transpile import CUSTOM_GLOBES, fast_rays, load_custom, params6
from test_supplied_lensmap_host_only import assert_same_state, state
from test_transpile import perturbed

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VALID, TINT_NONE = 0x80000000, 7


def lens_rays(fe, w, h):
    """[h, w, 3] float32: lens_inverse at each pixel of a build ((lx - w/2) * scale, -(ly - h/2) * scale), narrowed to
    float32, the zero vector where it returns nil; None when the lens has no lens_inverse"""
    s = fe.scale
    rays = np.zeros((h, w, 3), np.float32)
    for ly in range(h):
        y = -(ly - h // 2) * s
        for lx in range(w):
            st, r = fe.lens_inverse((lx - w // 2) * s, y)
            if st == -2:
                return None
            assert st in (0, 1), (fe.lens_name, lx, ly, st)
            if st == 1:
                rays[ly, lx] = r
    return rays


def map_state(fe):
    idx, tint = fe.lensmap()
    return {"idx": idx, "tint": tint, "packed": fe.lensmap_packed(), "display": fe.display(), "mapped": fe.mapped_pixels,
            "digest": fe.plan_digest(), "numplates": fe.numplates, "upload": fe.upload_bytes_per_frame}


def build_then_raymap(fe, w, h, ps):
    """(the build's state, the ray map's state) of the current lens and globe, or None for a forward-only lens"""
    fe.build_lensmap(w, h, ps, threads=1)
    want = map_state(fe)
    rays = lens_rays(fe, w, h)
    if rays is None:
        return None
    fe.set_raymap(rays, ps)
    assert fe.build_info.startswith("ray map, host"), fe.build_info
    return want, map_state(fe)


def test_every_inverse_lens_on_every_globe_equals_the_build_and_the_reference(host):
    lm = np.load(os.path.join(G, "lensmaps_small.npz"))
    meta = json.load(open(os.path.join(G, "meta_small.json")))
    W, H, PS = 128, 96, 48
    checked = 0
    for key in sorted(meta):   # the golden order: later globes see the plate slots earlier ones left
        g, l = key.split("__")
        host.command(f"f_globe {g}")
        host.command(f"f_lens {l}")
        r = build_then_raymap(host, W, H, PS)
        if r is None:
            continue
        want, got = r
        assert_same_state(want, got)
        assert np.array_equal(got["idx"], lm[key + "__idx"]), key
        assert np.array_equal(got["tint"], lm[key + "__tint"]), key
        assert got["display"] == meta[key]["display"], key
        assert host.scale == meta[key]["scale"], key
        checked += 1
    assert checked >= 40, checked


@pytest.mark.parametrize("globe", ["cube", "fast", "trism"])
def test_rubix_grids_and_odd_sizes_equal_the_build(host, globe):
    """another f_rubixgrid, rubix on, an odd screen and plate size"""
    from conftest import ALL_LENSES

    host.set_rubix(True)
    host.set_rubixgrid(4, 3.0, 2.0)
    for lens in ALL_LENSES[::3]:
        host.command(f"f_globe {globe}")
        host.command(f"f_lens {lens}")
        r = build_then_raymap(host, 97, 64, 37)
        if r is not None:
            assert_same_state(*r)


# ---- adversarial rays against the reference rule -------------------------------------------------------------------

def f32dot(a, b):
    return np.float32(np.float32(a[0] * b[0]) + np.float32(a[1] * b[1])) + np.float32(a[2] * b[2])


def ref_entry(ray, slots, numplates, ps, grid, plate_of=None):
    """The reference's rule for one float32 ray, written out: VectorNormalize, ray_to_plate_index (argmax of float dot
    products widened to double, or the globe's globe_plate), ray_to_plate_uv in double, (int) truncation, the rubix
    grid.  Returns the packed entry a single-pass map gives the pixel."""
    r = np.array(ray, np.float32)
    ln = np.float32(np.float32(r[0] * r[0]) + np.float32(r[1] * r[1])) + np.float32(r[2] * r[2])
    ln = np.float32(math.sqrt(float(ln))) if not math.isnan(ln) else ln
    if ln:
        inv = np.float32(1) / ln
        r = np.array([r[0] * inv, r[1] * inv, r[2] * inv], np.float32)
    if plate_of is None:
        best, best_dp = 0, -2.0
        for i in range(numplates):
            dp = float(f32dot(r, slots[i][0:3]))
            if dp > best_dp:
                best, best_dp = i, dp
    else:
        best = plate_of(float(r[0]), float(r[1]), float(r[2]))
        if best < 0 or best >= 6:
            return TINT_NONE << 28
    p = slots[best]
    x, y, z = float(f32dot(p[3:6], r)), float(f32dot(p[6:9], r)), float(f32dot(p[0:3], r))
    t = math.tan(float(np.float32(p[9]) / np.float32(2)))
    dist = 0.5 / t if t else math.inf
    u = (x / z if z else (math.copysign(math.inf, x) * math.copysign(1, z) if x and not math.isnan(x) else math.nan)) * dist + 0.5
    v = ((-y) / z if z else (math.copysign(math.inf, -y) * math.copysign(1, z) if y and not math.isnan(y) else math.nan)) * dist + 0.5
    if not (0 <= u <= 1 and 0 <= v <= 1):
        return TINT_NONE << 28
    px, py = int(u * ps), int(v * ps)
    if not (0 <= px < ps and 0 <= py < ps):
        return TINT_NONE << 28
    numcells, cell, pad = grid
    block = pad + cell
    unit_px = ps / (numcells * block + pad)
    ongrid = math.fmod(px / unit_px, block) < pad or math.fmod(py / unit_px, block) < pad
    return VALID | ((TINT_NONE if ongrid else best) << 28) | (best * ps * ps + px + py * ps)


def u_one_rays(slots, numplates, ps):
    """float32 rays a few ulps either side of each plate's right edge u = 1 (u * ps reaching ps is unmapped)"""
    out = []
    for plate in range(numplates):
        f, rt, up = (slots[plate][k:k + 3].astype(np.float64) for k in (0, 3, 6))
        t = math.tan(float(np.float32(slots[plate][9]) / np.float32(2)))
        for a in np.linspace(-0.9, 0.9, 7):
            base = f + rt * t + up * a * t     # u = 1 at the plate's right edge
            for k in range(-6, 7):
                ray = (base * (1 + k * 2.0 ** -24)).astype(np.float32)
                out.append(ray)
    return np.array(out, np.float32)


def adversarial_rays(slots, numplates, ps):
    inf, nan, tiny, den = np.inf, np.nan, np.float32(1e-45), np.float32(1e-40)
    special = [[0, 0, 0], [-0.0, 0, 0], [0, -0.0, -0.0], [nan, 0, 1], [0, nan, 0], [nan, nan, nan], [inf, 0, 0], [-inf, 0, 0],
               [inf, inf, 1], [inf, -inf, 0], [0, 0, -inf], [tiny, 0, 0], [0, den, 0], [den, den, den], [tiny, -tiny, tiny],
               [1e38, 0, 0], [1e38, 1e38, 1e38], [-1e38, 1, 0], [3e38, 3e38, 0],
               [1, 1, 0], [1, 0, 1], [0, 1, 1], [1, 1, 1], [-1, -1, -1], [1, -1, 1], [-1, 1, -1], [1, 1, -1],   # cube edges, corners
               [1, 0, 0], [0, 1, 0], [0, 0, 1], [-1, 0, 0], [0, -1, 0], [0, 0, -1], [2, 2, 0], [1e-20, 1e-20, 0]]
    rng = np.random.default_rng(3)
    rand = rng.normal(size=(400, 3)) * rng.choice([1e-30, 1e-3, 1.0, 1e20], size=(400, 1))
    return np.vstack([np.array(special, np.float32), rand.astype(np.float32), u_one_rays(slots, numplates, ps), fast_rays()[:300]])


@pytest.mark.parametrize("globe", ["cube", "cube_corner", "cube_edge", "tetra", "trism", "fast"])
def test_adversarial_rays_follow_the_reference_rule(host, globe):
    ps = 64
    host.command("f_globe cube")   # the slots beyond this globe's plates: the cube's
    slots = np.zeros((6, 11), np.float32)
    slots[:6] = host.plates()
    host.command(f"f_globe {globe}")
    pl = host.plates()
    slots[: len(pl)] = pl
    rays = adversarial_rays(slots, len(pl), ps)
    n = len(rays)
    w = 50
    h = -(-n // w)
    field = np.zeros((h * w, 3), np.float32)
    field[:n] = rays
    with np.errstate(all="ignore"):
        host.set_raymap(field.reshape(h, w, 3), ps)
        got = host.lensmap_packed().reshape(-1)
        plate_of = None
        if globe == "fast":
            plate_of = lambda x, y, z: host.globe_plate(x, y, z)[1]   # noqa: E731 (the interpreter's answer)
        want = np.array([ref_entry(r, slots, len(pl), ps, GRID, plate_of) for r in field], np.uint32)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, (globe, [(field[i].tolist(), hex(got[i]), hex(want[i])) for i in bad[:5]])
    assert 0 < (got & VALID).astype(bool).sum() < n


# ---- the ray-map kernel's text behind the CPU shim -------------------------------------------------------------------

RUN_RAYMAP = r"""
extern "C" void run_lt_raymap(const LtParams *P, const float *rays, unsigned *map, unsigned *flagged, unsigned *nflagged, unsigned cap) {
    blockDim.x = 256; blockDim.y = blockDim.z = 1;
    const size_t npix = (size_t)P->width * P->height;
    for (unsigned bx = 0; (size_t)bx * 256 < npix; ++bx)
        for (unsigned t = 0; t < 256; ++t) {
            blockIdx.x = bx; blockIdx.y = blockIdx.z = 0; threadIdx.x = t;
            lt_raymap(*P, rays, map, flagged, nflagged, cap);
        }
}
"""


@pytest.mark.parametrize("scale", [0, 1 << 20])   # 0 = host libm, else libm results off by up to 3*scale ulp
@pytest.mark.parametrize("globe", ["cube", "fast", "stale", "nan_huge", "latlon"])
def test_emulated_raymap_kernel_equals_the_host_path(host, tmp_path, globe, scale):
    w, h, ps = 96, 64, 40
    host.set_rubixgrid(*GRID)
    if globe in CUSTOM_GLOBES:
        slots = load_custom(host, globe)
    else:
        host.command("f_globe cube")
        slots = np.zeros((6, 11), np.float32)
        slots[:6] = host.plates()
        host.command(f"f_globe {globe}")
        slots[: host.numplates] = host.plates()
        host.command("f_lens panini")
    host.build_lensmap(w, h, ps, threads=1)   # the scale, for params6
    rng = np.random.default_rng(11)
    rays = rng.normal(size=(h * w, 3)).astype(np.float32)
    fr = fast_rays()
    rays[: min(len(fr), h * w)] = fr[: h * w]
    rays[::97] = 0
    rays = rays.reshape(h, w, 3)
    host.set_raymap(rays, ps)
    want = host.lensmap_packed().reshape(-1)

    src = host.lens_source(raymap=True)
    assert ("#define LT_HAS_GLOBE_PLATE 1" in src) == (globe != "cube")
    assert "lt_entry" not in src, "the ray-map unit holds no lens"
    if scale:
        src = perturbed(src, scale)
    lib = build_lib(src, RUN_RAYMAP, str(tmp_path / f"rm_{globe}_{scale}"))
    p = params6(host, w, h, ps, slots)
    got = np.zeros(h * w, np.uint32)
    flagged = np.zeros(h * w, np.uint32)
    n = ctypes.c_uint(0)
    lib.run_lt_raymap(ctypes.byref(p), rays.ctypes.data_as(ctypes.c_void_p), got.ctypes.data_as(ctypes.c_void_p),
                      flagged.ctypes.data_as(ctypes.c_void_p), ctypes.byref(n), ctypes.c_uint(h * w))
    flagged = flagged[: n.value]
    if globe == "cube":
        assert n.value == 0, "argmax globes raise no flag"
    if globe == "nan_huge":
        assert n.value > 0
    assert (got[flagged] == TINT_NONE << 28).all(), "flagged pixels are written unmapped"
    keep = np.ones(h * w, bool)
    keep[flagged] = False
    bad = np.nonzero((got != want) & keep)[0]
    assert bad.size == 0, (globe, scale, bad.size, [(hex(got[i]), hex(want[i])) for i in bad[:4]])


def test_raymap_source_flavours(bb, host):
    host.command("f_globe cube")
    plain = host.lens_source(raymap=True)
    cuda = host.lens_source(cuda=True, raymap=True)
    assert "lt_raymap" in plain and "lt_raymap" in cuda
    assert plain.startswith("#include <math.h>") and "#define LT_FN static __device__" in cuda
    assert "LT_HAS_GLOBE_PLATE 1" not in cuda
    host.command("f_globe fast")
    assert host.lens_source(cuda=True, raymap=True).startswith(host.lens_source(cuda=True, globe_plate=True))
    from test_globe_plate_transpile import REFUSED_GLOBES

    host.load_globe("t", REFUSED_GLOBES[0][0])
    with pytest.raises(bb.BlinkyError, match="booleans"):
        host.lens_source(raymap=True)


# ---- refusals and state ----------------------------------------------------------------------------------------------

def test_refusals_change_nothing(bb, host):
    lib = bb.load_library()
    fresh = bb.Fisheye(device=None)
    try:
        rays = np.zeros((8, 8, 3), np.float32)
        assert lib.blinky_set_raymap(fresh._ctx, 8, 8, 0, rays.ctypes.data) == bb.E_STATE, "no globe yet"
    finally:
        fresh.close()
    host.command("f_globe cube")
    host.command("f_lens stereographic")
    host.command("f_fov 200")
    W, H, ps = 96, 64, 32
    host.build_lensmap(W, H, ps, threads=1)
    rays = lens_rays(host, W, H)
    host.set_raymap(rays, ps)
    before = state(host)
    buf = np.zeros(3 * W * H + 1, np.float32)
    cases = [("NULL rays", W, H, ps, None), ("misaligned", W, H, ps, buf.ctypes.data + 2), ("width 0", 0, H, ps, rays.ctypes.data),
             ("height < 0", W, -1, ps, rays.ctypes.data), ("platesize too large", W, H, 6689, rays.ctypes.data)]
    for what, w, h, p, ptr in cases:
        assert lib.blinky_set_raymap(host._ctx, w, h, p, ptr) == bb.E_INVALID, what
        assert_same_state(before, state(host))
    assert lib.blinky_set_raymap_device(host._ctx, W, H, ps, rays.ctypes.data, None) == bb.E_NODEVICE
    # a globe_plate that raises an error: E_SCRIPT, nothing changes
    host.load_globe("boom", CUSTOM_GLOBES["fractions"].replace("if x > 0.2 then return 1.5 end", "if x > 0.2 then error('boom') end"))
    before = state(host)
    host.clear_log()
    assert lib.blinky_set_raymap(host._ctx, W, H, ps, rays.ctypes.data) == bb.E_SCRIPT
    assert "boom" in host.log
    assert_same_state(before, state(host))
    # 6 * 6688^2 < 2^28 is the largest plate size a build takes, whatever the globe
    host.command("f_globe cube")
    host.set_raymap(np.zeros((2, 3, 3), np.float32), 6688)
    assert host.platesize == 6688 and host.mapped_pixels == 0


def test_state_after_a_raymap(host):
    W, H, ps = 96, 64, 32
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.command("f_fov 180")
    host.build_lensmap(W, H, ps, threads=1)
    scale = host.scale
    rays = lens_rays(host, W, H)
    host.command("f_lens hammer")   # a lens change, consumed by the ray map
    assert host.needs_rebuild(W, H, ps)
    host.set_raymap(rays, ps)
    assert not host.needs_rebuild(W, H, ps) and host.needs_rebuild(W, H, ps + 1)
    assert host.scale == scale and host.lens_name == "hammer"
    assert (host.width, host.height, host.platesize) == (W, H, ps)
    # platesize 0 is min(width, height)
    host.set_raymap(rays)
    assert host.platesize == H
    # the same rays through another globe give that globe's build
    host.command("f_globe trism")
    host.set_raymap(rays, ps)
    got = map_state(host)
    host.command("f_lens panini")
    host.build_lensmap(W, H, ps, threads=1)
    assert host.scale == scale
    assert_same_state(map_state(host), got)


def test_the_stale_slot_globe_equals_its_build(host):
    W, H, ps = 120, 80, 48
    for name in ("stale", "fractions", "nan_huge", "mutable", "latlon"):
        load_custom(host, name)
        r = build_then_raymap(host, W, H, ps)
        assert_same_state(*r)
        if name == "stale":
            assert host.numplates == 2 and max(r[1]["display"]) == 1
            assert (r[1]["idx"] >= 2 * ps * ps).any(), "entries on the stale slots index beyond numplates * ps^2"
