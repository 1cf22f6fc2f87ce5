"""The Lua -> C++/CUDA lens translator (blinky_b200/csrc/lua_transpile.cpp) and the device
lensmap builder built on it (SURVEY section 8f rank 1).

CPU suite: the translated lens is compiled with g++ (same libm as the interpreter) and must
reproduce the interpreter's lens_inverse BIT FOR BIT; that pins the translator.  The CUDA
flavour of the same source must compile for sm_90a with NVRTC (no GPU needed for that).

GPU suite: blinky_build_lensmap(threads=0) evaluates the lens on the GPU; the finished
lensmap must equal the all-interpreter build for every translatable lens."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from conftest import ALL_GLOBES, ALL_LENSES

WRAP = r"""
extern "C" int lt_eval(double x, double y, const LtPlate *plates, int np, double *r, unsigned *flag) {
    Ctx c; c.flag = 0; c.steps = 0; c.plates = plates; c.numplates = np;
    lt_init_mut(c);
    LtD o[3];
    bool ok = lt_entry(c, x, y, o);
    if (ok) for (int i = 0; i < 3; ++i) { r[i] = o[i].v; r[3 + i] = o[i].e; lt_f32(c, o[i]); }
    *flag = c.flag;
    return ok ? 1 : 0;
}
"""

WRAP_FWD = r"""
extern "C" int lt_eval_fwd(double a0, double a1, double a2, double *r, unsigned *flag) {
    Ctx c; c.flag = 0; c.steps = 0; c.plates = 0; c.numplates = 0;
    lt_init_mut(c);
    LtD o[2];
    bool ok = lt_entry(c, a0, a1, a2, o);
    if (ok) for (int i = 0; i < 2; ++i) { r[i] = o[i].v; r[2 + i] = o[i].e; }
    *flag = c.flag;
    return ok ? 1 : 0;
}
"""

# lenses that must translate (closed-form and iterative alike); the rest of the shipped set is
# forward-only (no lens_inverse) or uses nil tests (debug) and takes the interpreter
TRANSLATABLE = ["cube", "cubestereo", "cylinder", "eckert4", "equirect", "fahey", "fisheye1", "fisheye2", "gallstereo",
                "gumby", "hammer", "mercator", "miller", "mollweide", "panini", "quincuncial", "rectilinear",
                "stereographic", "vandergrinten", "winkeltripel"]


def _points(n_random=700):
    W, H = 41, 31
    pts = [((lx - W // 2) * 0.11, -(ly - H // 2) * 0.11) for ly in range(H) for lx in range(W)]
    rng = np.random.default_rng(7)
    pts += [tuple(rng.uniform(-4, 4, 2)) for _ in range(n_random)]
    return pts


def _compile_host(src, path, wrap=WRAP):
    cpp = path + ".cpp"
    with open(cpp, "w") as f:
        f.write(src + wrap)
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    # -fno-builtin: g++ would fold libm calls on constants (sinh(2.0)) with MPFR, i.e. correctly rounded,
    # which is not always what glibc returns at run time
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fno-builtin", "-shared", "-fPIC", "-o", path + ".so", cpp],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:3000]
    lib = ctypes.CDLL(path + ".so")
    if wrap is WRAP:
        lib.lt_eval.argtypes = [ctypes.c_double, ctypes.c_double, ctypes.c_void_p, ctypes.c_int,
                                ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint)]
    else:
        lib.lt_eval_fwd.argtypes = [ctypes.c_double] * 3 + [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint)]
    return lib


@pytest.mark.parametrize("lens", TRANSLATABLE)
def test_translated_lens_is_bit_identical_to_the_interpreter(host, tmp_path, lens):
    host.command("f_globe cube")
    host.command(f"f_lens {lens}")
    lib = _compile_host(host.lens_source(cuda=False), str(tmp_path / lens))
    pl = host.plates()
    plates = np.zeros((6, 10), np.float32)
    plates[: len(pl), :9] = pl[:, :9]
    plates[: len(pl), 9] = pl[:, 10]
    out = (ctypes.c_double * 8)()
    flag = ctypes.c_uint()
    flagged = 0
    pts = _points()
    for x, y in pts:
        st, ray = host.lens_inverse(x, y)
        st2 = lib.lt_eval(x, y, plates.ctypes.data, len(pl), out, ctypes.byref(flag))
        assert st == st2, (lens, x, y)
        if st == 1:  # compare the bit patterns: NaN == NaN, -0.0 != 0.0
            assert struct.pack("3d", *ray) == struct.pack("3d", out[0], out[1], out[2]), (lens, x, y, ray, list(out[:3]))
        flagged += bool(flag.value)
    # the error bounds must not degenerate into "everything is uncertain"
    assert flagged <= 0.12 * len(pts), (lens, flagged, len(pts))


FORWARD_LENSES = [l for l in ALL_LENSES if l not in ("debug", "quincuncial")]  # every shipped lens_forward
FORWARD_ONLY = ["eckert1", "eckert5", "gins8", "kavrayskiy7", "larrivee", "polyconic", "sinusoidal", "wagner6", "winkel1", "winkel2"]


@pytest.mark.parametrize("lens", FORWARD_LENSES)
def test_translated_lens_forward_is_bit_identical_to_the_interpreter(host, tmp_path, lens):
    host.command("f_globe cube")
    host.command(f"f_lens {lens}")
    lib = _compile_host(host.lens_source(cuda=False, forward=True), str(tmp_path / lens), WRAP_FWD)
    rng = np.random.default_rng(11)
    rays = rng.normal(size=(900, 3))
    rays /= np.linalg.norm(rays, axis=1, keepdims=True)
    rays = rays.astype(np.float32).astype(np.float64)  # the builder feeds float32 rays
    rays = np.vstack([rays, [[0, 0, 1], [0, 0, -1], [1, 0, 0], [0, 1, 0], [0, -1, 0], [-1, 0, 0]]])
    out = (ctypes.c_double * 4)()
    flag = ctypes.c_uint()
    for rx, ry, rz in rays:
        st, xy = host.lens_forward(rx, ry, rz)
        st2 = lib.lt_eval_fwd(rx, ry, rz, out, ctypes.byref(flag))
        assert st == st2, (lens, rx, ry, rz)
        if st == 1:
            assert struct.pack("2d", *xy) == struct.pack("2d", out[0], out[1]), (lens, rx, ry, rz, xy, list(out[:2]))


def test_untranslatable_lenses_say_why(bb, host):
    host.command("f_globe cube")
    host.command("f_lens debug")
    with pytest.raises(bb.BlinkyError, match="nil"):
        host.lens_source()
    host.command("f_lens eckert1")  # forward-only
    with pytest.raises(bb.BlinkyError, match="no lens_inverse"):
        host.lens_source()
    for src, why in [
        ("function lens_inverse(x,y) local s = 'a' .. 'b' return x,y,1 end", "string"),
        ("function lens_inverse(x,y) local f = function() return 1 end return x,y,f() end", "closures"),
        ("local function r(n) if n < 1 then return 1 end return r(n-1) end function lens_inverse(x,y) return x,y,r(3) end", "recursive"),
        ("function lens_inverse(x,y) for k,v in pairs({}) do end return x,y,1 end", "for"),
        ("function lens_inverse(x,y,z) return x,y,1 end", "exactly"),
        ("function lens_inverse(x,y) print(x) return x,y,1 end", "print"),
        ("function lens_inverse(x,y) return x,y,math.random() end", "unsupported|resolve"),
        ("function lens_inverse(x,y) local t = x > 0 and 1 or 2 return x,y,t end", "and"),
        ("function lens_inverse(x,y) return x,y end", "three"),
    ]:
        host.load_lens("t", src)
        with pytest.raises(bb.BlinkyError, match=why):
            host.lens_source()


STATEFUL = """
local k = 2.5
local calls, memo = 0
function lens_inverse(x, y)
  calls = calls + 1
  if memo ~= y then memo = y end
  local t = {x, y, k}
  t[3] = t[3] * calls
  return latlon_to_ray(t[2] * 0.5 + memo * 0.5, t[1] + t[3] - k)
end"""


def test_script_level_state_is_per_pixel(host, tmp_path):
    """a lens that caches in script-level variables (like eckert4) translates: the variables
    become per-pixel state initialised from their values at translation time"""
    host.command("f_globe cube")
    host.load_lens("t", STATEFUL)
    src = host.lens_source()
    assert "c.mg[0]" in src and "c.mg[1]" in src
    lib = _compile_host(src, str(tmp_path / "t"))
    out = (ctypes.c_double * 8)()
    flag = ctypes.c_uint()
    for x, y in [(0.25, -0.5), (1.0, 0.3)]:
        host.load_lens("t", STATEFUL)  # back to the initial script-level values (calls == 0)
        st, want = host.lens_inverse(x, y)
        assert st == 1
        assert lib.lt_eval(x, y, None, 0, out, ctypes.byref(flag)) == 1
        assert struct.pack("3d", *want) == struct.pack("3d", out[0], out[1], out[2])


def test_cuda_flavour_of_every_lens_compiles_for_sm90a(bb, host):
    """NVRTC cross-compiles without a GPU; a missing libnvrtc is a skip, a compile error is a failure"""
    host.command("f_globe cube")
    compiled = 0
    for lens in ALL_LENSES:
        host.command(f"f_lens {lens}")
        for forward in (False, True):
            try:
                src = host.lens_source(cuda=True, forward=forward)
            except bb.BlinkyError:
                continue  # no such function, or outside the subset (covered elsewhere)
            assert "__device__" in src
            try:
                size = host.compile_lens(forward=forward)
            except bb.BlinkyError as e:
                if "NVRTC not found" in str(e):
                    pytest.skip(str(e))
                raise
            assert size > 1000, (lens, forward)
            compiled += 1
    assert compiled == len(TRANSLATABLE) + len(FORWARD_LENSES)


def test_threads_zero_without_gpu_uses_the_interpreter(host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.build_lensmap(96, 64, 32, threads=0)
    assert host.build_info.startswith("host")
    a = host.lensmap_packed().copy()
    host.build_lensmap(96, 64, 32, threads=1)
    assert np.array_equal(a, host.lensmap_packed())


# ----------------------------------------------------------------------------- GPU


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("lens", TRANSLATABLE)
def test_device_built_lensmap_equals_interpreter_build(bb, fe, lens):
    total = undecided = 0
    for globe, (w, h, ps), zoom, rubix in [("cube", (320, 200, 128), None, False), ("tetra", (257, 131, 96), "f_fov 200", True)]:
        fe.command(f"f_globe {globe}")
        fe.command(f"f_lens {lens}")
        if zoom:
            fe.command(zoom)
        fe.set_rubix(rubix)
        try:
            fe.build_lensmap(w, h, ps, threads=0)
        except bb.BlinkyError:
            # e.g. a zoom the lens cannot do: must fail identically on the host
            with pytest.raises(bb.BlinkyError):
                fe.build_lensmap(w, h, ps, threads=-1)
            continue
        info = fe.build_info
        assert info.startswith("device:"), (lens, globe, info)
        dev_idx, dev_tint = fe.lensmap()
        dev_disp = fe.display()
        fe.build_lensmap(w, h, ps, threads=-1)
        assert fe.build_info.startswith("host")
        idx, tint = fe.lensmap()
        assert np.array_equal(dev_idx, idx), (lens, globe, int((dev_idx != idx).sum()), info)
        assert np.array_equal(dev_tint, tint), (lens, globe, info)
        assert dev_disp == fe.display()
        undecided += int(info.split()[1])
        total += w * h
    assert undecided <= 0.12 * max(total, 1), (lens, undecided, total)


@pytest.mark.gpu
def test_device_build_every_shipped_lens_and_globe(bb, fe):
    """whatever the lens: threads=0 gives the interpreter's lensmap (device path or fallback)"""
    w, h, ps = 200, 120, 64
    ways = {}
    for globe in ALL_GLOBES:
        for lens in ALL_LENSES:
            fe.command(f"f_globe {globe}")
            fe.command(f"f_lens {lens}")
            try:
                fe.build_lensmap(w, h, ps, threads=0)
                ok = True
            except bb.BlinkyError:
                ok = False
            a = fe.lensmap_packed().copy()
            way = fe.build_info.split(":")[0].split(" ")[0]
            try:
                fe.build_lensmap(w, h, ps, threads=-1)
                ok2 = True
            except bb.BlinkyError:
                ok2 = False
            assert ok == ok2, (globe, lens)
            assert np.array_equal(a, fe.lensmap_packed()), (globe, lens, way)
            ways[way] = ways.get(way, 0) + 1
    assert ways.get("device", 0) >= len(TRANSLATABLE) * (len(ALL_GLOBES) - 1)


@pytest.mark.gpu
def test_device_build_full_size_matches_golden_c1(bb, fe):
    """BASELINE C1 (640x480 cube panini fov 180) built on the device == golden lensmap of the compiled reference"""
    import json

    G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    fe.command("f_globe cube")
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    fe.build_lensmap(640, 480, 256, threads=0)
    assert fe.build_info.startswith("device:")
    idx, tint = fe.lensmap()
    c1 = np.load(os.path.join(G, "c1.npz"))
    assert np.array_equal(idx, c1["idx"]) and np.array_equal(tint, c1["tint"])


@pytest.mark.gpu
@pytest.mark.parametrize("lens", FORWARD_ONLY)
def test_device_forward_builder_equals_interpreter_build(bb, fe, lens):
    """forward-only lenses: grid points on the GPU, quads rasterised on the GPU in the reference's
    writer order (last writer wins, tints stick) == the host's serial scanline builder"""
    for globe, (w, h, ps), rubix in [("cube", (320, 200, 96), False), ("tetra", (200, 131, 64), True)]:
        fe.command(f"f_globe {globe}")
        fe.command(f"f_lens {lens}")
        fe.set_rubix(rubix)
        fe.clear_log()
        fe.build_lensmap(w, h, ps, threads=0)
        info = fe.build_info
        assert info.startswith("device (forward):"), (lens, globe, info)
        dev_idx, dev_tint = fe.lensmap()
        dev_disp, dev_log = fe.display(), fe.log
        fe.clear_log()
        fe.build_lensmap(w, h, ps, threads=1)
        assert fe.build_info.startswith("host")
        idx, tint = fe.lensmap()
        assert np.array_equal(dev_idx, idx), (lens, globe, int((dev_idx != idx).sum()), info)
        assert np.array_equal(dev_tint, tint), (lens, globe, info)
        assert dev_disp == fe.display()
        assert dev_log == fe.log  # the "%d > maxdiff" console messages, in order


@pytest.mark.gpu
def test_device_forward_builder_with_nil_results(bb, fe):
    """lens_forward returning nil leaves stale row-buffer values behind in the reference; the device
    replays that, including the px == 0 `continue` that also skips the next slot"""
    src = """
    map = "lens_forward"
    max_fov = 360
    max_vfov = 180
    lens_width = 2*pi
    lens_height = pi
    onload = "f_contain"
    function lens_forward(x, y, z)
      local lat, lon = ray_to_latlon(x, y, z)
      if lat > 0.9 or (lon > 0.5 and lon < 0.7) or x*x < 0.0004 then
        return nil
      end
      return lon, lat
    end
    """
    for globe, (w, h, ps) in [("cube", (256, 128, 64)), ("trism", (199, 100, 48))]:
        fe.command(f"f_globe {globe}")
        fe.load_lens("holes", src)
        fe.clear_log()
        fe.build_lensmap(w, h, ps, threads=0)
        assert fe.build_info.startswith("device (forward):"), fe.build_info
        a = fe.lensmap_packed().copy()
        log_a = fe.log
        fe.clear_log()
        fe.build_lensmap(w, h, ps, threads=1)
        assert np.array_equal(a, fe.lensmap_packed()), int((a != fe.lensmap_packed()).sum())
        assert log_a == fe.log


# ----------------------------------------------------------------------------- soundness of the error bounds
#
# On the GPU the only arithmetic that may differ from the host is libm.  That is emulated here on
# the CPU: in a second build of the same translation every libm result is moved by a pseudo-random
# -3..+3 ulp ("some other libm").  Wherever that build raises no risk flag, its outcome must be the
# exact one: same nil/values status and the same float32 ray.  (Flagged points are the interpreter's.)

EXACT_LT_FN = """LT_FN LtD lt_fn(double r, double prop) {
    /* identical inputs and a NaN / infinite result (domain error, overflow): the same on both sides */
    if (prop == 0.0 && !(fabs(r) <= 1.79769313486231570815e308)) return LtD(r);
    return LtD(r, prop + LT_KU * fabs(r));
}"""

PERTURBED_LT_FN = """LT_FN LtD lt_fn(double r, double prop) {
    if (prop == 0.0 && !(fabs(r) <= 1.79769313486231570815e308)) return LtD(r);
    union { double d; unsigned long long u; } b;
    b.d = r;
    const unsigned long long h = (b.u ^ (b.u >> 29)) * 0x9E3779B97F4A7C15ull;
    const long long k = ((long long)((h >> 40) % 7ull) - 3) * PERT_SCALE;   /* -3 .. +3 (x PERT_SCALE) ulp */
    const unsigned long long frac = b.u & 0x000FFFFFFFFFFFFFull;
    if (r != 0.0 && frac > 8ull * PERT_SCALE && frac < 0x000FFFFFFFFFFFFFull - 8ull * PERT_SCALE) b.u += k;
    return LtD(b.d, prop + LT_KU * fabs(b.d));
}"""


EXACT_LT_FN_EDGE = """LT_FN LtD lt_fn_edge(double r, double prop, bool edge) {
    if (edge && fabs(r) < 0x1p-1022) return LtD(r, prop + LT_KU * 0x1p-1022);
    if (edge && fabs(r) > 0x1.ffffffffffff0p1023) return LtD(r, LT_INF);
    return lt_fn(r, prop);
}"""

# the range edges as another libm may round them: an underflowed 0 becomes the smallest subnormal, a subnormal moves
# by up to 3 of its ulps, and an overflowed inf becomes the largest double (lt_fn moves every other result)
PERTURBED_LT_FN_EDGE = """LT_FN LtD lt_fn_edge(double r, double prop, bool edge) {
    if (edge && fabs(r) < 0x1p-1022) {
        union { double d; unsigned long long u; } b;
        b.d = r;
        const unsigned long long h = (b.u ^ (b.u >> 29)) * 0x9E3779B97F4A7C15ull;
        const long long k = (long long)((h >> 40) % 4ull);   /* 0 .. 3 ulp of 2^-1074 away from 0 */
        b.u = (b.u & 0x8000000000000000ull) | ((b.u & 0x7FFFFFFFFFFFFFFFull) + k);
        if (r == 0.0) b.u |= 1ull;
        return LtD(b.d, prop + LT_KU * 0x1p-1022);
    }
    if (edge && fabs(r) > 0x1.ffffffffffff0p1023) return LtD(fabs(r) > 1.79769313486231570815e308 ? copysign(1.79769313486231570815e308, r) : r, LT_INF);
    return lt_fn(r, prop);
}"""


def perturbed(src, scale=1):
    """scale > 1 magnifies both the libm disagreement and the per-call bound by the same factor: the
    propagation rules hold to all orders, so they must hold at any scale, and at 2^20 ulp the rare
    events (a float32 rounding boundary inside the error interval) become frequent enough to be tested."""
    assert EXACT_LT_FN in src and EXACT_LT_FN_EDGE in src, "lt_fn / lt_fn_edge changed: update the test's copy"
    assert "#define LT_KU (8.0 * LT_U)" in src
    src = src.replace("#define LT_KU (8.0 * LT_U)", f"#define PERT_SCALE {scale}LL\n#define LT_KU (8.0 * PERT_SCALE * LT_U)")
    return src.replace(EXACT_LT_FN, PERTURBED_LT_FN).replace(EXACT_LT_FN_EDGE, PERTURBED_LT_FN_EDGE)


def f32bits(vals):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(vals, np.float64).astype(np.float32).tobytes()


def check_bounds_sound(host, lib, pts, what):
    out = (ctypes.c_double * 8)()
    flag = ctypes.c_uint()
    decided = 0
    for x, y in pts:
        st, ray = host.lens_inverse(x, y)
        st2 = lib.lt_eval(x, y, None, 0, out, ctypes.byref(flag))
        if flag.value:
            continue  # the interpreter decides this pixel
        decided += 1
        assert st == st2, (what, x, y, st, st2)
        if st == 1:
            assert f32bits(ray) == f32bits([out[0], out[1], out[2]]), (what, x, y, ray, list(out[:6]))
    return decided


@pytest.mark.parametrize("scale", [1, 1 << 20])
@pytest.mark.parametrize("lens", [l for l in TRANSLATABLE if l not in ("cube", "cubestereo")])  # those two use plate_to_ray
def test_error_bounds_are_sound_under_a_different_libm(host, tmp_path, lens, scale):
    host.command("f_globe cube")
    host.command(f"f_lens {lens}")
    lib = _compile_host(perturbed(host.lens_source(cuda=False), scale), str(tmp_path / f"{lens}{scale}"))
    pts = _points(2500)
    decided = check_bounds_sound(host, lib, pts, (lens, scale))
    assert decided >= (0.4 if scale == 1 else 0.05) * len(pts), (lens, scale, decided, len(pts))


EDGES = """
function lens_inverse(x, y)
  local t = math.exp(x * 200 - 745)      -- 0, a subnormal or a normal number around x = 0
  local s = math.exp(709.78 + y * 0.01)  -- finite below y = 0.27, inf above
  local p = 2 ^ (1023.99 + x * 0.01)     -- the same for pow
  local lat, lon = y * 0.3, x * 0.3
  if t > 0 then lon = lon + 0.1 end
  if s < math.huge then lat = lat - 0.05 end
  if p == math.huge then lon = lon - 0.2 end
  return latlon_to_ray(lat, lon)
end"""


@pytest.mark.parametrize("scale", [1, 1 << 20])
def test_error_bounds_are_sound_at_the_range_edges(host, tmp_path, scale):
    """exp and pow at their underflow and overflow thresholds, where another libm may give 0 for a subnormal or inf
    for the largest double: the perturbed build moves those results too, and every decision it leaves unflagged must
    still be the interpreter's"""
    host.command("f_globe cube")
    host.load_lens("edges", EDGES)
    lib = _compile_host(perturbed(host.lens_source(cuda=False), scale), str(tmp_path / f"edges{scale}"))
    xs = np.concatenate([np.linspace(-0.05, 0.3, 71), [-4.0, -1.0, 1.0, 4.0]])
    ys = np.concatenate([np.linspace(0.2, 0.35, 61), [-3.0, 0.0, 3.0]])
    pts = [(x, y) for x in xs for y in ys]
    decided = check_bounds_sound(host, lib, pts, ("edges", scale))
    assert decided >= (0.3 if scale == 1 else 0.1) * len(pts), (scale, decided, len(pts))
