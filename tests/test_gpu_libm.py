"""The device's double libm, through the translated lenses' own wrappers, against the interpreter's libm.

A device lensmap build is the interpreter's bit for bit because every libm result carries a bound: lt_fn
charges LT_KU * |r| (8 ulp) per call, exact arguments giving a NaN or infinite result count as identical,
and exp, sinh, cosh, pow and atan2 get an absolute floor below the normal range and an infinite bound at
the overflow threshold (lt_fn_edge, blinky_b200/csrc/lua_transpile.cpp).  blinky_probe_math runs those
wrappers on the GPU from the prelude text every lens unit starts with, so this file checks the claim
itself, per function, on ~10^6 arguments: lens-domain sweeps, random bit patterns over the whole
double range, and the hard cases (the doubles nearest k pi/2, huge trig arguments, the edges of asin,
acos and log, zeros, subnormals, infinities and NaN, the overflow and underflow thresholds, atan2's
signed zeros and infinities, pow of negative bases and of bases near 1).

The host side is glibc through ctypes: what the interpreter's std::sin, std::pow, ... call.  Asserted:
  * where the device reports e == 0 the host's result is bitwise the same (NaN matches NaN);
  * otherwise, for a finite device result, |v_dev - v_host| <= e;
  * the operations DESIGN section 4b calls IEEE-identical (sqrt, fmod, floor, ceil, trunc, modf, /,
    float narrowing, int conversion) are bitwise the host's.
On a subset (20 k per function plus every hard case) both sides are measured in ulps against mpmath,
and the device is held to the CUDA Math API's documented maximum errors (CUDA_DOC_ULP), or to the measured
maximum where the H100 exceeds them (CUDA_MEASURED_OVER_DOC).  The table
printed at the end is the one in DESIGN section 4b."""
import ctypes
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
mpmath = pytest.importorskip("mpmath")

pytestmark = pytest.mark.gpu

# Maximum ulp errors of the double-precision functions, CUDA C++ Programming Guide, appendix "Mathematical
# Functions", table "Double-Precision Mathematical Standard Library Functions with Maximum ULP Error" (CUDA 12.9),
# with the IEEE operations at 0.  logb (Lua's math.log(x, base)) is log(x) / log(base): two roundings of
# documented functions, so it has no entry of its own.
CUDA_DOC_ULP = {"sin": 2, "cos": 2, "tan": 2, "asin": 2, "acos": 2, "atan": 2, "atan2": 2, "exp": 1, "log": 1, "log10": 1,
                "sinh": 2, "cosh": 1, "tanh": 1, "pow": 2}
# Where the H100 (CUDA 12.9 NVRTC, sm_90a) measured more on this file's arguments, the measured maximum: the
# prelude's 8 ulp per call still covers it, which the contract assertions check.  tan: 2.33 ulp at 2103.296...
# (tan = -8.7e12, next to a pole); log10: 1.35 ulp at 3504.22...; cosh: 1.15 ulp at 10.78...; tanh: 1.08 ulp at 0.5438...
CUDA_MEASURED_OVER_DOC = {"tan": 2.33, "log10": 1.36, "cosh": 1.15, "tanh": 1.08}
LIBM_OPS = ["sin", "cos", "tan", "asin", "acos", "atan", "atan2", "exp", "log", "log10", "logb", "sinh", "cosh", "tanh", "pow"]
IEEE_OPS = ["sqrt", "fmod", "floor", "ceil", "trunc", "modf", "div", "f32", "int"]

DMAX = np.finfo(np.float64).max
TINY = np.finfo(np.float64).smallest_subnormal
SPECIAL = np.array([0.0, -0.0, TINY, -TINY, 2.0**-1022, -(2.0**-1022), 2.0**-1030, -(2.0**-1050), np.inf, -np.inf, np.nan,
                    1.0, -1.0, DMAX, -DMAX])

_libm = ctypes.CDLL("libm.so.6")
for _f in ("sin", "cos", "tan", "asin", "acos", "atan", "exp", "log", "log10", "sinh", "cosh", "tanh", "sqrt", "floor", "ceil",
           "trunc"):
    getattr(_libm, _f).restype = ctypes.c_double
    getattr(_libm, _f).argtypes = [ctypes.c_double]
for _f in ("atan2", "pow", "fmod"):
    getattr(_libm, _f).restype = ctypes.c_double
    getattr(_libm, _f).argtypes = [ctypes.c_double, ctypes.c_double]
_libm.modf.restype = ctypes.c_double
_libm.modf.argtypes = [ctypes.c_double, ctypes.POINTER(ctypes.c_double)]


def host(op, a, b):
    """the interpreter's result (minilua calls std:: functions, i.e. glibc; math.log(x, base) is lmathlib's)"""
    n = len(a)
    v = np.empty(n)
    e = np.zeros(n)
    al, bl = a.tolist(), b.tolist()
    if op in ("atan2", "pow", "fmod"):
        f = getattr(_libm, op)
        v[:] = [f(x, y) for x, y in zip(al, bl)]
    elif op == "logb":
        log, log10 = _libm.log, _libm.log10
        with np.errstate(all="ignore"):
            v[:] = [log10(x) if y == 10.0 else float(np.float64(log(x)) / np.float64(log(y))) for x, y in zip(al, bl)]
    elif op == "div":
        with np.errstate(all="ignore"):
            v[:] = a / b
    elif op == "f32":
        with np.errstate(all="ignore"):
            v[:] = a.astype(np.float32).astype(np.float64)
    elif op == "int":
        v[:] = np.trunc(a) + 0.0   # (int) has no -0
    elif op == "modf":
        ip = ctypes.c_double()
        f = _libm.modf
        for i, x in enumerate(al):
            v[i] = f(x, ctypes.byref(ip))
            e[i] = ip.value
    else:
        f = getattr(_libm, op)
        v[:] = [f(x) for x in al]
    return v, e


def same_bits(x, y):
    """bitwise equal, any NaN equal to any NaN"""
    return (x.view(np.uint64) == y.view(np.uint64)) | (np.isnan(x) & np.isnan(y))


# ----------------------------------------------------------------------------- arguments


def _near(x, k):
    """x and its k neighbouring doubles on each side"""
    x = np.atleast_1d(np.asarray(x, np.float64))
    out = [x]
    up, dn = x.copy(), x.copy()
    for _ in range(k):
        up, dn = np.nextafter(up, np.inf), np.nextafter(dn, -np.inf)
        out += [up, dn]
    return np.concatenate(out)


def _bits(rng, n):
    x = rng.integers(0, 2**64, n, dtype=np.uint64).view(np.float64)
    return x[np.isfinite(x)]


def _pi_multiples(rng):
    ks = np.concatenate([np.arange(1, 8193), rng.integers(8193, 2**20 + 1, 8000)])
    with mpmath.workprec(200):
        pi2 = mpmath.pi / 2
        xs = np.array([float(int(k) * pi2) for k in ks])
    return _near(np.concatenate([xs, -xs]), 1)


def _huge(rng):
    j = rng.integers(20, 1024, 6000)
    return np.ldexp(rng.uniform(1.0, 2.0, 6000), j) * rng.choice([-1.0, 1.0], 6000)


def arguments(op, seed=1):
    """(sweep + random bits, hard cases): each a pair of arrays (a, b)"""
    rng = np.random.default_rng(seed + LIBM_OPS.index(op) if op in LIBM_OPS else seed + 100 + IEEE_OPS.index(op))
    N = 1 << 19
    if op in ("sin", "cos", "tan"):
        sweep = np.concatenate([rng.uniform(-4 * np.pi, 4 * np.pi, 2 * N), _bits(rng, N)])
        hard = np.concatenate([_pi_multiples(rng), _huge(rng), SPECIAL])
    elif op in ("asin", "acos"):
        sweep = np.concatenate([rng.uniform(-1, 1, 2 * N), _bits(rng, N // 4), rng.uniform(-1e-3, 1e-3, N // 2)])
        k = np.arange(0, 6000) * 2.0**-53
        hard = np.concatenate([1 - k, -1 + k, _near([1.0, -1.0, 0.5, -0.5], 8), SPECIAL])
    elif op == "atan":
        sweep = np.concatenate([rng.uniform(-100, 100, 2 * N), np.exp(rng.uniform(-700, 700, N // 2)), _bits(rng, N // 2)])
        hard = np.concatenate([_near([1.0, -1.0, 1e16, 2.0**-27], 8), SPECIAL])
    elif op == "atan2":
        t = rng.uniform(-np.pi, np.pi, 2 * N)
        r = np.exp(rng.uniform(-30, 30, 2 * N))
        y, x = r * np.sin(t), r * np.cos(t)
        by, bx = _bits(rng, N // 2), _bits(rng, N // 2)
        m = min(len(by), len(bx))
        sweep = (np.concatenate([y, by[:m]]), np.concatenate([x, bx[:m]]))
        sv = np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -1.5, TINY, -TINY, DMAX, -DMAX, np.nan])
        gy, gx = np.meshgrid(sv, sv)
        base = rng.uniform(0.1, 100, 4000) * rng.choice([-1.0, 1.0], 4000)
        ratio = _near(base, 4)
        hard = (np.concatenate([gy.ravel(), ratio, -ratio, np.full(4, 1e-300), np.full(4, TINY)]),
                np.concatenate([gx.ravel(), np.tile(base, 9), np.tile(base, 9), [1e300, -1e300, 1e10, 3.0], [1e300, 1.0, -1.0, 1e-300]]))
        return sweep, hard
    elif op in ("exp", "sinh", "cosh", "tanh"):
        sweep = np.concatenate([rng.uniform(-40, 40, 2 * N), rng.uniform(-750, 750, N // 2), _bits(rng, N // 2)])
        edges = {"exp": [709.782712893384, -708.3964185322641, -745.1332191019411, -744.4400719213812],
                 "sinh": [710.4758600739439, -710.4758600739439], "cosh": [710.4758600739439, -710.4758600739439],
                 "tanh": [19.06154746539849, -19.06154746539849, 0.55]}[op]
        hard = np.concatenate([_near(edges, 8), SPECIAL])
    elif op in ("log", "log10"):
        sweep = np.concatenate([rng.uniform(0, 1e4, 2 * N), 1 + rng.uniform(-1e-3, 1e-3, N // 2), np.abs(_bits(rng, N // 2))])
        k = np.arange(1, 6000) * 2.0**-52
        hard = np.concatenate([1 + k, 1 - k / 2, _near([1.0, 10.0, 100.0, 0.1], 8), -_bits(rng, 1000), SPECIAL])
    elif op == "logb":
        xs = np.exp(rng.uniform(-50, 50, N))
        bases = rng.choice([2.0, 10.0, 0.5, math.e, 3.0, 1.0 + 1e-9], N)
        sweep = (xs, bases)
        hard = (np.concatenate([SPECIAL, SPECIAL, _near([1.0, 10.0, 1024.0], 8)]),
                np.concatenate([np.full(len(SPECIAL), 2.0), np.full(len(SPECIAL), 10.0), np.full(51, 10.0)]))
        return sweep, hard
    elif op == "pow":
        base = rng.uniform(0, 10, 2 * N)
        ex = np.where(rng.random(2 * N) < 0.5, rng.choice([0.5, 2.0, 3.0, -1.0, 1 / 3], 2 * N), rng.uniform(-10, 10, 2 * N))
        ba, bb_ = _bits(rng, N // 2), rng.uniform(-60, 60, N // 2)
        m = min(len(ba), len(bb_))
        sweep = (np.concatenate([base, ba[:m]]), np.concatenate([ex, bb_[:m]]))
        hb, he = [], []
        for b in (2.0, 10.0, 0.5, 1.5, 7.25, 1e-3, 1e10):   # y log2 b = 1024 (overflow), -1022 and -1074 (underflow)
            for target in (1024.0, -1022.0, -1074.0):
                y = _near(target / math.log2(b), 8)
                hb.append(np.full(len(y), b))
                he.append(y)
        neg = -rng.uniform(0.1, 50, 3000)
        ints = rng.integers(-60, 61, 3000).astype(np.float64)
        hb += [neg, neg, _near([1.0], 16), _near([1.0], 16), _near([-1.0], 4)]
        he += [ints, ints + 0.5, np.full(33, 1e15), np.full(33, -3e17), np.full(9, 2.0**60)]
        sv = np.array([0.0, -0.0, np.inf, -np.inf, 1.0, -1.0, 0.5, -2.0, 3.0, np.nan, TINY, DMAX])
        gb, ge = np.meshgrid(sv, sv)
        hb.append(gb.ravel())
        he.append(ge.ravel())
        return sweep, (np.concatenate(hb), np.concatenate(he))
    elif op == "sqrt":
        sweep = np.concatenate([rng.uniform(0, 1e4, N), _bits(rng, N)])
        hard = SPECIAL
    elif op in ("fmod", "div"):
        a, b = _bits(rng, N), _bits(rng, N)
        m = min(len(a), len(b))
        a2, b2 = rng.uniform(-1e3, 1e3, N), rng.uniform(-10, 10, N)
        sweep = (np.concatenate([a[:m], a2]), np.concatenate([b[:m], b2]))
        gy, gx = np.meshgrid(SPECIAL, SPECIAL)
        return sweep, (gy.ravel(), gx.ravel())
    elif op in ("floor", "ceil", "trunc", "modf"):
        sweep = np.concatenate([rng.uniform(-1e6, 1e6, N), _bits(rng, N)])
        hard = np.concatenate([_near(np.arange(-8, 9) * 0.5, 2), _near([2.0**52, 2.0**53, -(2.0**52)], 2), SPECIAL])
    elif op == "f32":
        f = rng.integers(0, 2**32, N, dtype=np.uint64).astype(np.uint32).view(np.float32)
        f = f[np.isfinite(f)].astype(np.float64)
        mid = (f + np.nextafter(f.astype(np.float32), np.float32(np.inf)).astype(np.float64)) / 2   # float rounding ties
        fmax = float(np.finfo(np.float32).max)
        sweep = np.concatenate([_bits(rng, N), mid[np.isfinite(mid)]])
        hard = np.concatenate([_near([fmax, fmax * (1 + 2.0**-25), 2.0**-149, 2.0**-150, 2.0**-126], 4), SPECIAL])
    elif op == "int":
        sweep = rng.uniform(-(2.0**31) + 1, 2.0**31 - 1, N)
        hard = np.concatenate([_near([0.0, 0.5, -0.5, 2.0**31 - 1, -(2.0**31)], 2)[2:], [0.0, -0.0]])
        hard = hard[(hard > -(2.0**31) - 1) & (hard < 2.0**31)]
    else:
        raise KeyError(op)
    return (sweep, np.zeros_like(sweep)), (hard, np.zeros_like(hard))


# ----------------------------------------------------------------------------- ulps against mpmath

_MP_FN = {
    "sin": mpmath.sin, "cos": mpmath.cos, "tan": mpmath.tan, "asin": mpmath.asin, "acos": mpmath.acos, "atan": mpmath.atan,
    "exp": mpmath.exp, "log": mpmath.log, "log10": mpmath.log10, "sinh": mpmath.sinh, "cosh": mpmath.cosh, "tanh": mpmath.tanh,
}


def _true(op, x, y):
    """the exact value (mpf) or None where it is not a finite real"""
    if not (math.isfinite(x) and math.isfinite(y)):
        return None
    X, Y = mpmath.mpf(x), mpmath.mpf(y)
    if op in ("asin", "acos") and abs(x) > 1 or op in ("log", "log10") and x <= 0:
        return None
    if op == "atan2":
        if x == 0.0:   # atan2(+-0, x): +-0 or +-pi by the sign of the zero, which mpmath does not keep
            return None if y == 0.0 else mpmath.pi * (0 if y > 0 else math.copysign(1.0, x))
        return mpmath.atan2(X, Y)
    if op == "logb":
        return mpmath.log(X) / mpmath.log(Y) if x > 0 and y > 0 and y != 1 else None
    if op == "pow":
        if x == 0:
            return None
        if x < 0:
            return (-1) ** int(y) * mpmath.power(-X, Y) if y == math.floor(y) else None
        return mpmath.power(X, Y)
    return _MP_FN[op](X)


def _ulps(got, true):
    """|got - true| in ulps of the true value's binade; an inf for a finite true value counts as 2^1024"""
    if abs(true) >= 2**1024 or math.isnan(got):
        return None
    if math.isinf(got):
        got = math.copysign(2.0**1023, got) * 2
    ulp = mpmath.ldexp(1, max(int(mpmath.floor(mpmath.log(abs(true), 2))) if true != 0 else -1074, -1022) - 52)
    return float(abs(mpmath.mpf(got) - true) / ulp)


def ulp_errors(op, a, b, dev, hst):
    worst_dev = worst_host = 0.0
    where = None
    with mpmath.workprec(160):
        for x, y, d, h in zip(a.tolist(), b.tolist(), dev.tolist(), hst.tolist()):
            t = _true(op, x, y)
            if t is None:
                continue
            ud, uh = _ulps(d, t), _ulps(h, t)
            if ud is not None and ud > worst_dev:
                worst_dev, where = ud, (x, y, d, h)
            if uh is not None:
                worst_host = max(worst_host, uh)
    return worst_dev, worst_host, where


def _dist_ulps(x, y):
    """|x - y| in ulps of y (finite, same class)"""
    ok = np.isfinite(x) & np.isfinite(y)
    u = np.spacing(np.abs(np.where(ok, y, 0.0)))
    return float(np.max(np.abs(x - y)[ok] / u[ok], initial=0.0))


# ----------------------------------------------------------------------------- the test

TABLE = {}


@pytest.fixture(scope="module")
def fe(bb, cuda_device):
    f = bb.Fisheye(device=cuda_device)
    yield f
    f.close()
    if TABLE:
        print("\nop      args      e==0   max|dev-host| ulp   dev ulp (mpmath)   host ulp (mpmath)   notes")
        for op, row in TABLE.items():
            print(f"{op:6s} {row['n']:8d} {row['exact']:8d} {row['dh']:17.3g} {row['dev']:18.3g} {row['host']:19.3g}   {row['notes']}")


def _device(fe, op, a, b):
    A = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    B = torch.from_numpy(np.ascontiguousarray(b)).cuda()
    v, e = fe.probe_math(op, A, B)
    return v.cpu().numpy(), e.cpu().numpy()


@pytest.mark.parametrize("op", LIBM_OPS + IEEE_OPS)
def test_device_libm_meets_the_bounds_the_prelude_charges(fe, op):
    (sa, sb), (ha, hb) = arguments(op)
    a, b = np.concatenate([sa, ha]), np.concatenate([sb, hb])
    dv, de = _device(fe, op, a, b)
    hv, he = host(op, a, b)
    ident = same_bits(dv, hv)
    notes = []
    if op in IEEE_OPS:
        bad = ~ident | (op == "modf") & ~same_bits(de, he)
        assert not bad.any(), (op, [(a[i], b[i], dv[i], hv[i], de[i], he[i]) for i in np.flatnonzero(bad)[:8]])
        TABLE[op] = dict(n=len(a), exact=len(a), dh=0.0, dev=0.0, host=0.0, notes="bitwise")
        return
    exact = de == 0
    bad = exact & ~ident
    assert not bad.any(), (op, "e == 0 but the host differs",
                           [(a[i], b[i], dv[i], hv[i]) for i in np.flatnonzero(bad)[:8]])
    with np.errstate(all="ignore"):
        checked = ~exact & np.isfinite(dv) & np.isfinite(de)
        over = checked & ~(np.abs(dv - hv) <= de)
    assert not over.any(), (op, "|dev - host| > e", [(a[i], b[i], dv[i], hv[i], de[i]) for i in np.flatnonzero(over)[:8]])
    # what the range edges gave: results the relative bound cannot cover, and how they differ
    tiny = checked & (np.abs(dv) < 2.0**-1022) & ~ident
    inf_edge = ~np.isfinite(de) & np.isfinite(a) & np.isfinite(b)
    if tiny.any():
        notes.append(f"{int(tiny.sum())} subnormal/zero results differ (max {np.max(np.abs(dv - hv)[tiny]) / TINY:.0f} x 2^-1074)")
    if inf_edge.any():
        notes.append(f"{int(inf_edge.sum())} infinite bounds from finite arguments, {int((inf_edge & ~ident).sum())} of them differ")
    # ulps against mpmath: a subset of the sweep and every hard case
    rng = np.random.default_rng(5)
    pick = np.concatenate([rng.choice(len(sa), min(20000, len(sa)), replace=False), len(sa) + np.arange(len(ha))])
    worst_dev, worst_host, where = ulp_errors(op, a[pick], b[pick], dv[pick], hv[pick])
    TABLE[op] = dict(n=len(a), exact=int(exact.sum()), dh=_dist_ulps(dv, hv), dev=worst_dev, host=worst_host, notes="; ".join(notes))
    if op in CUDA_DOC_ULP:
        limit = max(CUDA_DOC_ULP[op], CUDA_MEASURED_OVER_DOC.get(op, 0))
        assert worst_dev <= limit + 1e-9, (op, "above the CUDA Math API's documented error (and the recorded maximum)", worst_dev, where)
