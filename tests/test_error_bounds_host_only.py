"""Every error-propagation rule of the translator's prelude against its mathematical claim.

A translated lens carries, next to each double, a bound `e` on how far the host's value may be from
the one computed here (transpile_prelude in blinky_b200/csrc/lua_transpile.cpp).  A rule such as
`operator/` or `lt_tan` takes inputs (v, e) and must bound |f(x') - r| for EVERY x' within e of v,
where r is the value the rule computed: not only to first order, because a chain of operations makes
input errors large compared with their distance to a pole (cancellation in `1 - cos(x)` is enough).
The decisions' x2 margin is not counted here, since errors compound along a chain.

The CPU flavour of the prelude is compiled with g++ (the flags test_transpile uses) behind one
`extern "C"` wrapper, so the test checks the code itself.  The true supremum over the input interval
(or box, for binary rules) comes from mpmath at 200 bits: endpoints or corners, interior critical
points and a dense grid.  An interval that reaches a pole, a domain edge or a region where the host
would produce NaN must give an infinite or NaN bound, which flags every decision that reads it."""
import ctypes
import math
import os
import subprocess

import mpmath
import pytest


WRAP_RULE = r"""
extern "C" int lt_rule(int op, double av, double ae, double bv, double be, double *out) {
    const LtD a(av, ae), b(bv, be);
    Ctx c; c.flag = 0; c.steps = 0; c.plates = 0; c.numplates = 0;
    LtD r;
    switch (op) {
        case 0: r = a / b; break;
        case 1: r = a * b; break;
        case 2: r = a + b; break;
        case 3: r = lt_sqrt(a); break;
        case 4: r = lt_sin(a); break;
        case 5: r = lt_cos(a); break;
        case 6: r = lt_tan(a); break;
        case 7: r = lt_asin(a); break;
        case 8: r = lt_acos(a); break;
        case 9: r = lt_atan(a); break;
        case 10: r = lt_atan2(a, b); break;
        case 11: r = lt_exp(a); break;
        case 12: r = lt_log(a); break;
        case 13: r = lt_log10(a); break;
        case 14: r = lt_logb(a, b); break;
        case 15: r = lt_sinh(a); break;
        case 16: r = lt_cosh(a); break;
        case 17: r = lt_tanh(a); break;
        case 18: r = lt_pow(a, b); break;
        case 19: r = lt_fmodD(c, a, b); break;
        case 20: r = lt_modD(c, a, b); break;
        default: return -1;
    }
    out[0] = r.v;
    out[1] = r.e;
    return (int)c.flag;
}
"""

mpmath.mp.prec = 200
MP = mpmath.mp
INF = math.inf


def _trunc(x):
    return MP.floor(x) if x >= 0 else MP.ceil(x)


def _pow(a, b):
    if a == 0:
        return MP.inf if b < 0 else MP.zero
    if a < 0 and b != MP.floor(b):
        return None  # NaN on the host
    return MP.power(a, b) if a > 0 else (-1) ** int(b) * MP.power(-a, b)


# name: (op, arity, f(x[, y]) on mpf (None = NaN on the host))
RULES = {
    "div": (0, 2, lambda a, b: a / b),
    "mul": (1, 2, lambda a, b: a * b),
    "add": (2, 2, lambda a, b: a + b),
    "sqrt": (3, 1, lambda x: MP.sqrt(x) if x >= 0 else None),
    "sin": (4, 1, MP.sin),
    "cos": (5, 1, MP.cos),
    "tan": (6, 1, MP.tan),
    "asin": (7, 1, lambda x: MP.asin(x) if abs(x) <= 1 else None),
    "acos": (8, 1, lambda x: MP.acos(x) if abs(x) <= 1 else None),
    "atan": (9, 1, MP.atan),
    "atan2": (10, 2, lambda y, x: MP.atan2(y, x)),
    "exp": (11, 1, MP.exp),
    "log": (12, 1, lambda x: MP.log(x) if x > 0 else None),
    "log10": (13, 1, lambda x: MP.log10(x) if x > 0 else None),
    "logb": (14, 2, lambda x, b: MP.log(x) / MP.log(b) if x > 0 and b > 0 and b != 1 else None),
    "sinh": (15, 1, MP.sinh),
    "cosh": (16, 1, MP.cosh),
    "tanh": (17, 1, MP.tanh),
    "pow": (18, 2, _pow),
    "fmod": (19, 2, lambda a, b: a - _trunc(a / b) * b if b != 0 else None),
    "mod": (20, 2, lambda a, b: a - MP.floor(a / b) * b if b != 0 else None),
}

HALF_PI = MP.pi / 2


def _contains(lo, hi, x):
    return lo <= x <= hi


def _singular(name, lo, hi, blo=None, bhi=None):
    """True when the interval (box) reaches a pole, a domain edge or a NaN region of the host's function"""
    if name in ("div", "fmod", "mod"):
        return _contains(blo, bhi, 0)
    if name == "sqrt":
        return lo < 0
    if name == "tan":
        return MP.floor(lo / MP.pi - MP.mpf(0.5)) != MP.floor(hi / MP.pi - MP.mpf(0.5))
    if name in ("asin", "acos"):
        return lo < -1 or hi > 1
    if name in ("log", "log10"):
        return lo <= 0
    if name == "logb":
        return lo <= 0 or blo <= 0 or _contains(blo, bhi, 1)
    if name == "atan2":  # (y, x): the box holds the origin or crosses the branch cut along the negative x axis
        return (_contains(lo, hi, 0) and _contains(blo, bhi, 0)) or (_contains(lo, hi, 0) and lo < hi and blo < 0)
    if name == "pow":
        exact_b = blo == bhi
        if exact_b and blo == MP.floor(blo):  # integer exponent: any base sign, a pole at 0 for negative ones
            return blo < 0 and _contains(lo, hi, 0)
        return lo <= 0 and not (exact_b and blo > 0 and lo == 0)
    return False


def _critical(name, lo, hi):
    """interior points where f' vanishes: a supremum of |f(x') - r| can sit there"""
    pts = []
    if name in ("sin", "cos"):
        off = HALF_PI if name == "sin" else 0
        k = MP.ceil((lo - off) / MP.pi)
        while off + k * MP.pi <= hi and len(pts) < 8:
            pts.append(off + k * MP.pi)
            k += 1
    if name == "cosh" and _contains(lo, hi, 0):
        pts.append(MP.zero)
    return pts


def _sup(name, f, r, lo, hi, blo=None, bhi=None, n=33):
    ts = [MP.mpf(i) / (n - 1) for i in range(n)]
    xs = [lo + (hi - lo) * t for t in ts] + _critical(name, lo, hi)
    if blo is None:
        pairs = [(x,) for x in xs]
    else:
        m = 17
        ys = [blo + (bhi - blo) * MP.mpf(i) / (m - 1) for i in range(m)]
        pairs = [(x, y) for x in xs[:: (n - 1) // (m - 1)] for y in ys]
        # the boundary densely: extremes of a harmonic atan2 sit there
        pairs += [(x, y) for x in xs for y in (blo, bhi)] + [(x, y) for x in (lo, hi) for y in ys]
    best = MP.zero
    for p in pairs:
        v = f(*p)
        if v is None:
            return MP.inf
        best = max(best, abs(v - r))
    return best


@pytest.fixture(scope="module")
def rule(tmp_path_factory, bb):
    h = bb.Fisheye(device=None)
    h.command("f_globe cube")
    h.load_lens("t", "function lens_inverse(x, y) return x, y, 1 end")
    src = h.lens_source(cuda=False)
    h.close()
    path = str(tmp_path_factory.mktemp("rules") / "rules")
    with open(path + ".cpp", "w") as f:
        f.write(src + WRAP_RULE)
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    # the flags of test_transpile._compile_host: the interpreter's own libm, no constant folding by MPFR
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fno-builtin", "-shared", "-fPIC", "-o", path + ".so", path + ".cpp"],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:3000]
    lib = ctypes.CDLL(path + ".so")
    lib.lt_rule.argtypes = [ctypes.c_int] + [ctypes.c_double] * 4 + [ctypes.POINTER(ctypes.c_double)]
    out = (ctypes.c_double * 2)()

    def call(name, av, ae, bv=0.0, be=0.0):
        flag = lib.lt_rule(RULES[name][0], av, ae, bv, be, out)
        assert flag >= 0
        return out[0], out[1], flag

    return call


REL = [2.0**-50, 2.0**-30, 2.0**-12, 0.125, 0.3, 0.5, 0.6, 0.8, 0.9, 0.99, 1.2, 2.0, 4.0]
NEAR = [0.01, 0.3, 0.6, 0.8, 0.9, 0.99, 1.2, 2.0]   # fractions of the distance to a singularity


def _unary_cases():
    c = []
    def add(name, vs, abs_e=(), near=None):
        for v in vs:
            es = [abs(v) * r for r in REL] if v != 0 else [2.0**-50, 2.0**-20, 0.1, 1.0]
            es += list(abs_e)
            if near is not None:
                d = near(v)
                es += [d * k for k in NEAR]
            c.extend((name, float(v), float(e)) for e in es if e > 0)
    pole = lambda v: float(min(abs(MP.mpf(v) - (HALF_PI + k * MP.pi)) for k in range(-6, 6)))
    add("sqrt", [1e-10, 0.25, 2.0, 1e10])
    add("sin", [0.0, 1.0, math.pi / 2, 100.0], abs_e=(0.5, 2.0, 7.0))
    add("cos", [0.0, 1.0, math.pi / 2, 100.0], abs_e=(0.5, 2.0, 7.0))
    add("tan", [0.3, 1.0, -2.5, 10.0, math.pi / 2 - 1e-3, math.pi / 2 - 1e-8, math.pi / 2, -math.pi / 2 + 0.01, 2.5 * math.pi - 1e-4],
        near=pole)
    edge = lambda v: 1.0 - abs(v)
    add("asin", [0.3, -0.7, 0.99, 1 - 2.0**-20, -1 + 1e-12], near=edge)
    add("acos", [0.3, -0.7, 0.99, 1 - 2.0**-20, -1 + 1e-12], near=edge)
    add("asin", [0.0, 1.0, -1.0])
    add("acos", [0.0, 1.0])
    add("atan", [0.0, 0.2, -1.0, 3.0, 1e8], abs_e=(0.5, 3.0))
    add("exp", [0.0, 1.0, -3.0, 20.0, -700.0, 700.0], abs_e=(2.0**-50, 2.0**-30, 1e-3, 0.1, 0.5, 0.9, 2.0))
    add("log", [1e-300, 1e-5, 0.5, 1.0, 1 + 2.0**-40, 3.0, 1e300], near=lambda v: v)
    add("log10", [1e-300, 1e-5, 0.5, 1.0, 3.0, 1e300], near=lambda v: v)
    for f in ("sinh", "cosh", "tanh"):
        add(f, [0.0, 0.5, -3.0, 20.0, -300.0], abs_e=(2.0**-50, 2.0**-30, 1e-3, 0.1, 0.5, 0.9, 2.0))
    return c


def _binary_cases():
    c = []
    errs = [0.0, 2.0**-40, 0.1, 0.5, 0.9, 0.99, 1.5]
    for name, pts in [("div", [(1.0, 2.0), (-3.5, -0.7), (1e-3, 1e-8), (0.0, 3.0), (5.0, 1.0)]),
                      ("mul", [(0.0, 0.0), (1.5, -2e-3), (1e5, 3.0), (0.0, 2.0)]),
                      ("add", [(1.0, -1.0), (3.0, 1e-9)]),
                      ("atan2", [(1.0, 1.0), (1e-3, -1.0), (-2.0, 0.5), (0.3, -1e-9), (0.0, 1.0), (5.0, 5.0), (-1e-12, -3.0)]),
                      ("logb", [(3.0, 2.0), (0.5, 0.5), (7.0, 1.001), (100.0, 10.0)]),
                      ("fmod", [(7.3, 2.0), (-7.3, 2.0), (1e-3, 3.0)]),
                      ("mod", [(7.3, 2.0), (-7.3, 2.0), (1e-3, -3.0)])]:
        for a, b in pts:
            for ra in errs:
                for rb in errs:
                    if ra == 0 and rb == 0:
                        continue
                    # relative to the operand, or to the other operand when the operand is 0
                    ea = ra * (abs(a) if a else abs(b))
                    eb = rb * (abs(b) if b else abs(a))
                    c.append((name, a, ea, b, eb))
    # pow: exact exponents of the shipped lenses and others, then both operands uncertain
    for base in (0.0, 0.5, 2.0, -1.5, 1e-3, 1 + 1e-9):
        for ex in (0.5, 2.0, 3.0, -1.0, 1 / 3, 2.5, -2.0):
            es = [r * abs(base) for r in REL] if base else [2.0**-50, 0.1, 1.0]
            c += [("pow", base, e, ex, 0.0) for e in es]
    for base in (0.5, 2.0, 1e-3, 7.0):
        for ex in (0.5, 2.0, -1.3, 40.0):
            for ra in (0.0, 2.0**-40, 0.1, 0.5, 0.9):
                for rb in (2.0**-40, 0.01, 0.1, 0.5):
                    c.append(("pow", base, ra * base, ex, rb * abs(ex)))
    return c


def _check(rule, name, av, ae, bv=None, be=None):
    r, e, flag = rule(name, av, ae, 0.0 if bv is None else bv, 0.0 if be is None else be)
    if flag:
        return None  # a decision inside the rule went to the interpreter
    lo, hi = MP.mpf(av) - MP.mpf(ae), MP.mpf(av) + MP.mpf(ae)
    blo = bhi = None
    if bv is not None:
        blo, bhi = MP.mpf(bv) - MP.mpf(be), MP.mpf(bv) + MP.mpf(be)
    if _singular(name, lo, hi, blo, bhi):
        return None if not math.isfinite(e) else f"{name}({av}±{ae}, {bv}±{be}): reaches a singularity, bound {e}"
    if not math.isfinite(r) or not math.isfinite(e):
        return None  # an infinite / NaN bound flags every decision; an infinite value is past this test
    f = RULES[name][2]
    sup = _sup(name, f, MP.mpf(r), lo, hi, blo, bhi)
    # (the bound is itself evaluated in double: a relative 2^-40 for its own rounding)
    if sup > MP.mpf(e) * (1 + MP.mpf(2) ** -40):
        return f"{name}({av}±{ae}, {bv}±{be}) = {r}: true sup {float(sup):.6g} > bound {e:.6g} (x{float(sup / e) if e else INF:.4g})"
    return None


def _run(rule, cases):
    bad = []
    for case in cases:
        name, av, ae = case[:3]
        why = _check(rule, name, av, ae, *case[3:])
        if why:
            bad.append(why)
    return bad


@pytest.mark.parametrize("name", ["sqrt", "sin", "cos", "tan", "asin", "acos", "atan", "exp", "log", "log10", "sinh", "cosh", "tanh"])
def test_unary_rule_bounds_the_true_change_to_all_orders(rule, name):
    cases = [c for c in _unary_cases() if c[0] == name]
    assert cases
    bad = _run(rule, cases)
    assert not bad, f"{len(bad)} of {len(cases)} cases:\n" + "\n".join(bad[:25])


@pytest.mark.parametrize("name", ["div", "mul", "add", "atan2", "logb", "pow", "fmod", "mod"])
def test_binary_rule_bounds_the_true_change_to_all_orders(rule, name):
    cases = [c for c in _binary_cases() if c[0] == name]
    assert cases
    bad = _run(rule, cases)
    assert not bad, f"{len(bad)} of {len(cases)} cases:\n" + "\n".join(bad[:25])


@pytest.mark.parametrize("name, av, ae, bv, be", [
    ("div", 1.0, 0.0, 1.0, 0.6), ("div", 1.0, 0.0, 1.0, 0.9), ("div", 1.0, 0.0, 1.0, 1.5),
    ("tan", 1.0, 0.6 * (math.pi / 2 - 1.0), None, None), ("tan", 1.0, 1.2 * (math.pi / 2 - 1.0), None, None),
    ("log", 1.0, 0.8, None, None), ("log", 1.0, 2.0, None, None), ("exp", 1.0, 2.0, None, None),
    ("sqrt", 1.0, 1.5, None, None), ("atan2", 0.1, 0.2, 0.1, 0.2), ("atan2", 1e-3, 1e-2, -1.0, 0.0),
    ("mul", 0.0, 1e-3, 0.0, 1e-3), ("asin", 0.9, 0.09, None, None), ("pow", 1.0, 0.8, 0.5, 0.0),
])
def test_known_weak_cases(rule, name, av, ae, bv, be):
    """the inputs where the first-order rules fell short of the truth (true/bound up to 10, or unbounded)"""
    assert _check(rule, name, av, ae, bv, be) is None


def test_exact_inputs_stay_exact(rule):
    """no rule may invent an error: exact operands give e == 0 (the decisions then need no interpreter)"""
    for name, a, b in [("div", 1.0, 3.0), ("mul", 0.1, 0.7), ("sqrt", 2.0, 0.0), ("sin", 0.0, 0.0), ("exp", 1.0, 0.0),
                       ("atan2", 0.0, 1.0), ("pow", 2.0, 0.5), ("pow", 0.0, 2.0), ("log", 1.0, 0.0), ("acos", 1.0, 0.0)]:
        r, e, _ = rule(name, a, 0.0, b, 0.0)
        if name in ("div", "mul", "sqrt") or r == 0.0:
            assert e == 0.0, (name, a, b, r, e)


def test_math_probe_unit_compiles_for_sm90a(bb):
    """blinky_probe_math with n = 0 compiles the probe unit (the lenses' prelude and the probe kernel) with NVRTC and the
    lens units' options, without a GPU; a missing libnvrtc is a skip, a compile error a failure"""
    import re
    header = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "blinky_b200.h")).read()
    block = header[header.index("BLINKY_PROBE_SIN = 0"):header.index("BLINKY_PROBE_COUNT")]
    names = [n.lower() for n in re.findall(r"BLINKY_PROBE_([A-Z0-9]+)\b", re.sub(r"/\*.*?\*/", "", block, flags=re.S))]
    assert tuple(names) == bb.Fisheye.PROBE_OPS   # the binding's op numbers are the header's
    h = bb.Fisheye(device=None)
    try:
        try:
            h.probe_math("sin")
        except bb.BlinkyError as e:
            if "NVRTC not found" in str(e):
                pytest.skip(str(e))
            raise
        with pytest.raises(bb.BlinkyError) as e:   # unknown op
            h._check(h._lib.blinky_probe_math(h._ctx, len(h.PROBE_OPS), None, None, None, None, 0, None))
        assert e.value.code == bb.E_INVALID
        with pytest.raises(bb.BlinkyError) as e:   # a host-only context runs nothing
            h._check(h._lib.blinky_probe_math(h._ctx, 0, 8, None, 8, 8, 1, None))
        assert e.value.code == bb.E_NODEVICE
    finally:
        h.close()


@pytest.mark.parametrize("name, av, bv", [
    ("exp", -745.2, None), ("exp", -745.1332191019411, None), ("exp", -744.5, None), ("exp", -708.5, None),
    ("exp", 709.782712893384, None), ("exp", 709.7827128933841, None), ("exp", 710.0, None),
    ("sinh", 710.4758600739439, None), ("sinh", -710.5, None), ("cosh", 710.4758600739439, None), ("cosh", -711.0, None),
    ("pow", 2.0, 1024.0), ("pow", 2.0, 1023.9999999999999), ("pow", 2.0, -1074.0), ("pow", 2.0, -1075.0), ("pow", 0.5, 1080.0),
    ("pow", -2.0, 1025.0), ("atan2", 1e-300, 1e300), ("atan2", -1e-300, 1e300),
])
def test_range_edges_get_bounds_another_libm_can_meet(rule, name, av, bv):
    """exact arguments at the overflow and underflow thresholds: a libm within a few ulp may give the largest double
    where another gives inf, or 0 where another gives the smallest subnormal.  LT_KU * |r| covers neither, so the
    bound must be infinite for a result within 16 ulp of the overflow threshold (inf included), and at least the
    smallest normal number's 8 ulp (8 * 2^-1074) for a result below the normal range (0 included)"""
    r, e, _ = rule(name, av, 0.0, 0.0 if bv is None else bv, 0.0)
    if abs(r) > float.fromhex("0x1.ffffffffffff0p1023"):
        assert e == INF, (name, av, bv, r, e)
    elif abs(r) < 2.0**-1022:
        assert e >= 8 * 2.0**-1074, (name, av, bv, r, e)
    else:   # (the largest finite exp, sinh, cosh and pow results are 20 ulp and more below the threshold)
        assert e >= 8 * 2.0**-52 * abs(r), (name, av, bv, r, e)


def test_exact_zeros_and_infinities_stay_exact(rule):
    """results the arguments make exact on every libm (IEEE 754 / C99 Annex F) keep e == 0: no decision on them goes
    to the interpreter"""
    for name, a, b in [("exp", -INF, 0.0), ("exp", INF, 0.0), ("sinh", 0.0, 0.0), ("sinh", -0.0, 0.0), ("pow", 0.0, 3.0),
                       ("pow", 0.0, -1.0), ("atan2", 0.0, 5.0), ("atan2", 3.0, INF), ("log", 0.0, 0.0), ("sin", 0.0, 0.0)]:
        r, e, _ = rule(name, a, 0.0, b, 0.0)
        assert e == 0.0, (name, a, b, r, e)
