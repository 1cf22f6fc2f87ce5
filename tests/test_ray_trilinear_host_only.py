"""The trilinear warp from a ray field (blinky_warp_device_rays_trilinear, Fisheye.warp_rays(filter="trilinear")) without a
GPU: the header functions of csrc/ray_texel.h (plate projection, footprint, level and weight, the pyramid's layout and the
positions on a level), compiled with g++ -ffp-contract=off behind tests/ray_trilinear_reference.py's shim as the kernel's
translation unit is with --fmad=false, against an independent numpy restatement; the binding's argument checks; the
refusal of a host-only context; and the kernel's instances in the built library and in its ptxas log.  The GPU path is
tests/test_gpu_ray_trilinear.py."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import ray_trilinear_reference as tr
from test_device_emulation import GRID
from test_ray_warp_host_only import ARGMAX_GLOBES, FakeCuda, matrices, params, turned
from test_raymap_host_only import adversarial_rays
from test_transpile import TRANSLATABLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, PS = 96, 64, 40


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return tr.compile_shim(tmp_path_factory.mktemp("ray_trilinear"))


# ---- the rule, restated in numpy ----------------------------------------------------------------------------------

def normalised(r):
    """normalize3 in float32: len = (float)sqrt((double)((x x + y y) + z z)), each component times 1 / len unless len is 0"""
    r = np.ascontiguousarray(r, np.float32).copy()
    f32 = np.float32
    with np.errstate(all="ignore"):
        ln = (r[..., 0] * r[..., 0] + r[..., 1] * r[..., 1]) + r[..., 2] * r[..., 2]
        ln = np.sqrt(ln.astype(np.float64)).astype(f32)
        inv = f32(1) / ln
        return np.where((ln != 0)[..., None], r * inv[..., None], r).astype(f32)


def dot(n, vec):
    a = np.asarray(vec, np.float32)
    with np.errstate(all="ignore"):
        return ((n[..., 0] * a[0] + n[..., 1] * a[1]) + n[..., 2] * a[2]).astype(np.float64)


def project(p, plate, n):
    """(usable, a, b) of normalised rays n [..., 3] onto plates `plate` (an int array of n's shape[:-1])"""
    x, y, z, uvd = (np.zeros(n.shape[:-1]) for _ in range(4))
    for i in range(p.numplates):
        sel = plate == i
        pl = p.plates[i]
        x[sel], y[sel], z[sel] = dot(n, pl.right)[sel], dot(n, pl.up)[sel], dot(n, pl.forward)[sel]
        uvd[sel] = p.uv_dist[i]
    ok = z > 0
    with np.errstate(all="ignore"):
        q = uvd * p.platesize / np.where(ok, z, 1.0)
        return ok, x * q, -y * q


def level(rho2, lmax):
    """(L, w) by the rule: rho = sqrt(rho2); the largest L <= lmax with 2^L <= rho (0 below 1 and for NaN); w"""
    rho = np.sqrt(np.asarray(rho2, np.float64))
    L = np.zeros(rho.shape, np.int64)
    with np.errstate(invalid="ignore"):
        for lv in range(1, lmax + 1):
            L = np.where(rho >= 2.0 ** lv, lv, L)
        frac = np.where(rho >= 1, rho / 2.0 ** L - 1, 0)
        w = np.where((rho >= 1) & (L < lmax), np.trunc(frac * 256), 0)
    return L, w.astype(np.int64)


def restated(p, field, M, lmax):
    """per pixel of field [h, w, 3] turned by M: (mapped, plate, rho2, L, w, u, v)"""
    h, w = field.shape[:2]
    t = field if M is None else turned(field, M)
    n = normalised(t)
    best = np.zeros((h, w), np.int64)
    best_dp = np.full((h, w), -2.0)
    for i in range(p.numplates):
        dp = dot(n, p.plates[i].forward)
        win = dp > best_dp
        best = np.where(win, i, best)
        best_dp = np.where(win, dp, best_dp)
    ok, a, b = project(p, best, n)   # (the same dot products as the plate's x, y, z)
    x, y, z, uvd = (np.zeros((h, w)) for _ in range(4))
    for i in range(p.numplates):
        sel = best == i
        pl = p.plates[i]
        x[sel], y[sel], z[sel] = dot(n, pl.right)[sel], dot(n, pl.up)[sel], dot(n, pl.forward)[sel]
        uvd[sel] = p.uv_dist[i]
    ps = p.platesize
    with np.errstate(all="ignore"):
        u = x / z * uvd + 0.5
        v = -y / z * uvd + 0.5
        inr = (u >= 0) & (u <= 1) & (v >= 0) & (v <= 1)
        uu, vv = np.where(inr, u, 0.0), np.where(inr, v, 0.0)
        mapped = inr & (np.trunc(uu * ps) < ps) & (np.trunc(vv * ps) < ps)

        def axis(fwd, back):
            """fwd / back: (exists, ray) shifted fields; the axis's da^2 + db^2, 0 where neither neighbour serves"""
            out = np.zeros((h, w))
            done = np.zeros((h, w), bool)
            for exists, nb in (fwd, back):
                okn, a1, b1 = project(p, best, nb)
                use = ~done & exists & okn
                out = np.where(use, (a1 - a) * (a1 - a) + (b1 - b) * (b1 - b), out)
                done |= use
            return out

        cols, rows = np.arange(w)[None, :], np.arange(h)[:, None]
        rx = axis((cols + 1 < w, np.roll(n, -1, axis=1)), (cols > 0, np.roll(n, 1, axis=1)))
        ry = axis((rows + 1 < h, np.roll(n, -1, axis=0)), (rows > 0, np.roll(n, 1, axis=0)))
        rho2 = np.where(ok, np.where(ry > rx, ry, rx), 0.0)
    L, wt = level(rho2, lmax)
    return mapped, best, rho2, L, wt, uu, vv


def positions(u, v, size):
    sx, sy = u * size - 0.5, v * size - 0.5
    x0, y0 = np.floor(sx), np.floor(sy)
    return x0.astype(np.int64), y0.astype(np.int64), np.trunc((sx - x0) * 256).astype(np.int64), np.trunc((sy - y0) * 256).astype(np.int64)


def same_double(a, b):
    """bitwise equal, every NaN equal to every NaN"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))


def assert_follows_the_rule(lib, p, field, M, what):
    """the shim's per-pixel values against the restatement; returns the shim's (s, rho2) of the mapped pixels"""
    h, w = field.shape[:2]
    sizes = tr.level_sizes(p.platesize)
    lmax = len(sizes) - 1
    s, rho2 = tr.header_trilinear(lib, p, M, field, lmax)
    mapped, plate, r2, L, wt, u, v = (a.reshape(-1) for a in restated(p, field, M, lmax))
    m = s[:, 0] == 1
    bad = np.nonzero(m != mapped)[0]
    assert bad.size == 0, (what, "mapped", bad.size, bad[:4].tolist())
    bad = np.nonzero(m & ((s[:, 1] != plate) | ~same_double(rho2, r2) | (s[:, 2] != L) | (s[:, 3] != wt)))[0]
    assert bad.size == 0, (what, "footprint", bad.size, [(s[i].tolist(), rho2[i], plate[i], r2[i], L[i], wt[i]) for i in bad[:4]])
    for col, lv in ((4, L), (8, np.minimum(L + 1, lmax))):
        size = np.asarray(sizes)[lv]
        want = np.stack(positions(u, v, size), axis=1)
        sel = m & (lv > L) if col == 8 else m
        bad = np.nonzero(sel & (s[:, col:col + 4] != want).any(axis=1))[0]
        assert bad.size == 0, (what, "positions", col, bad.size, [(s[i].tolist(), want[i].tolist()) for i in bad[:4]])
    assert ((s[m, 3] >= 0) & (s[m, 3] <= 255)).all() and ((s[m, 2] >= 0) & (s[m, 2] <= lmax)).all(), what
    return s[m], rho2[m]


# ---- the header against the restatement ---------------------------------------------------------------------------

def test_every_translatable_lens_turned(lib, host):
    host.command("f_globe cube")
    host.set_rubixgrid(*GRID)
    checked = 0
    levels, weights = set(), set()
    for lens in TRANSLATABLE:
        host.command(f"f_lens {lens}")
        host.command("f_fov 180")
        try:
            rays = host.raymap(W, H)
        except Exception:  # noqa: BLE001 — a zoom this lens cannot do
            continue
        for ps in (PS, 512):
            p = params(host, W, H, ps, GRID)
            for i, M in enumerate(matrices()):
                s, _ = assert_follows_the_rule(lib, p, rays, M, (lens, ps, i))
                levels.update(s[:, 2].tolist())
                weights.update(s[:, 3].tolist())
        checked += 1
    assert checked >= 15, checked
    assert {0, 1, 2, 3} <= levels, sorted(levels)
    assert len(weights) > 200, "the weights cover their range"


@pytest.mark.parametrize("globe", ARGMAX_GLOBES)
def test_argmax_globes(lib, host, globe):
    host.set_rubixgrid(*GRID)
    host.command(f"f_globe {globe}")
    host.command("f_lens panini")
    host.command("f_fov 180")
    rays = host.raymap(W, H)
    rng = np.random.default_rng(len(globe))
    rays.reshape(-1, 3)[::7] = rng.normal(size=rays.reshape(-1, 3)[::7].shape).astype(np.float32)
    p = params(host, W, H, 97, GRID)
    mapped = 0
    for i, M in enumerate(matrices(seed=len(globe))):
        mapped += len(assert_follows_the_rule(lib, p, rays, M, (globe, i))[0])
    assert mapped > 0


@pytest.mark.parametrize("globe", ARGMAX_GLOBES)
def test_adversarial_rays_and_missing_neighbours(lib, host, globe):
    """zeros, NaN, +-inf, subnormals, rays behind a plate and on plate edges, as a one-row field (no y neighbours), a
    one-column field (no x neighbours), a 1 x 1 field (none) and a block whose edges lack the forward neighbours"""
    host.set_rubixgrid(*GRID)
    host.command(f"f_globe {globe}")
    slots = np.zeros((6, 11), np.float32)
    pl = host.plates()
    slots[: len(pl)] = pl
    ps = 64
    rays = adversarial_rays(slots, len(pl), ps)
    fwd = np.asarray(pl[0][0:3], np.float32)
    extra = np.array([[-3e38, 3e38, 1], [-0.0, -0.0, 1], [1, -0.0, 0], [np.float32(1e-45), 1, 0], [1, 1, np.nan], -fwd, fwd,
                      fwd + np.float32(1e-7), fwd * np.float32(1e-30)], np.float32)
    rays = np.vstack([rays, extra])
    n = len(rays) - len(rays) % 4
    p = params(host, 50, 50, ps, GRID)
    for i, M in enumerate([None] + list(matrices(seed=3))):
        assert_follows_the_rule(lib, p, rays[None], M, (globe, i, "row"))
        assert_follows_the_rule(lib, p, rays[:, None], M, (globe, i, "column"))
        assert_follows_the_rule(lib, p, rays[:1][None], M, (globe, i, "1x1"))
        assert_follows_the_rule(lib, p, rays[:n].reshape(4, n // 4, 3), M, (globe, i, "block"))


def test_projection_behind_and_beside_the_plate(lib, host):
    """ray_plate_project: usable exactly when z > 0 (not for z = 0, -0, NaN), with a and b as restated"""
    host.command("f_globe cube")
    p = params(host, 8, 8, 97, GRID)
    pl = host.plates()
    rng = np.random.default_rng(1)
    rays = normalised(np.vstack([rng.normal(size=(500, 3)), [pl[0][3:6], -np.asarray(pl[0][0:3]), [0, 0, 0], [np.nan, 0, 1]]]).astype(np.float32))
    for plate in range(p.numplates):
        ok = np.zeros(len(rays), np.uint8)
        a, b = np.zeros(len(rays)), np.zeros(len(rays))
        lib.project(ctypes.byref(p), plate, np.ascontiguousarray(rays).ctypes.data, len(rays), ok.ctypes.data, a.ctypes.data, b.ctypes.data)
        wok, wa, wb = project(p, np.full(len(rays), plate), rays)
        assert np.array_equal(ok.astype(bool), wok)
        assert same_double(a[wok], wa[wok]).all() and same_double(b[wok], wb[wok]).all()
        assert 0 < wok.sum() < len(rays)


def test_footprint_takes_the_backward_neighbour_when_the_forward_one_fails(lib, host):
    """per axis: forward when it exists and projects usably, else backward, else 0; rho^2 = x unless y is greater"""
    host.command("f_globe cube")
    p = params(host, 8, 8, 97, GRID)
    fwd = np.asarray(host.plates()[0][0:3], np.float32)
    right = np.asarray(host.plates()[0][3:6], np.float32)
    n = normalised(fwd)
    near = normalised(fwd + np.float32(0.01) * right)
    far = normalised(fwd + np.float32(0.05) * right)
    behind = -fwd
    cases = [  # (xf, xb, yf, yb) or None, expected source: "xf", "xb", "yf", "yb", 0
        ((near, far, None, None), "xf"), ((behind, far, None, None), "xb"), ((None, far, None, None), "xb"), ((behind, behind, None, None), 0),
        ((None, None, None, None), 0), ((near, None, far, None), "yf"), ((far, None, near, None), "xf"), ((None, None, behind, near), "yb"),
    ]
    count = len(cases)
    nb = np.zeros((count, 4, 3), np.float32)
    has = np.zeros((count, 4), np.uint8)
    for i, (q, _) in enumerate(cases):
        for k, r in enumerate(q):
            if r is not None:
                nb[i, k], has[i, k] = r, 1
    out = np.zeros(count)
    plate = np.zeros(count, np.int32)
    lib.footprint(ctypes.byref(p), plate.ctypes.data, np.ascontiguousarray(np.repeat(n[None], count, 0)).ctypes.data, nb.ctypes.data,
                  has.ctypes.data, count, out.ctypes.data)
    _, a, b = project(p, np.zeros(1, np.int64), n[None])
    for i, (q, src) in enumerate(cases):
        if src == 0:
            assert out[i] == 0, i
            continue
        r = q[["xf", "xb", "yf", "yb"].index(src)]
        _, a1, b1 = project(p, np.zeros(1, np.int64), r[None])
        assert out[i] == (a1[0] - a[0]) ** 2 + (b1[0] - b[0]) ** 2 or out[i] == (a1[0] - a[0]) * (a1[0] - a[0]) + (b1[0] - b[0]) * (b1[0] - b[0]), i
        assert out[i] > 0


def test_level_and_weight_at_powers_of_four(lib):
    """rho^2 exactly 4^L and one ulp either side, for every lmax; 0, subnormal, inf and NaN"""
    vals = [0.0, 5e-324, 0.25, np.inf, np.nan, -0.0, 1e300]
    for L in range(15):
        x = 4.0 ** L
        vals += [np.nextafter(x, 0), x, np.nextafter(x, np.inf), x * 2.25, x * 3.99]
    rho2 = np.array(vals, np.float64)
    for lmax in range(14):
        got_L = np.zeros(len(rho2), np.int32)
        got_w = np.zeros(len(rho2), np.int32)
        lib.level(rho2.ctypes.data, len(rho2), lmax, got_L.ctypes.data, got_w.ctypes.data)
        L, w = level(rho2, lmax)
        assert np.array_equal(got_L, L) and np.array_equal(got_w, w), (lmax, [(v, a, b, c, d) for v, a, b, c, d in zip(rho2, got_L, L, got_w, w) if a != b or c != d][:4])
    # one ulp below 4^L is level L - 1 with weight 255; 4^L itself is level L with weight 0
    lv = np.zeros(3, np.int32)
    wt = np.zeros(3, np.int32)
    x = np.array([np.nextafter(16.0, 0), 16.0, np.nan])
    lib.level(x.ctypes.data, 3, 5, lv.ctypes.data, wt.ctypes.data)
    assert lv.tolist() == [1, 2, 0] and wt.tolist() == [255, 0, 0]


@pytest.mark.parametrize("ps, lmax", [(1, 0), (2, 1), (3, 2), (97, 7), (2048, 11), (6688, 13)])
def test_pyramid_sizes(lib, ps, lmax):
    sizes, offs, total, raw = tr.pyramid_layout(ps, 6)
    assert len(sizes) - 1 == lmax and sizes[-1] == 1
    assert tr.header_pyramid(lib, ps, 6) == (lmax, sizes, offs, total)
    assert total % 256 == 0 and total - raw < 256
    for nplates in (1, 4, 5):
        assert tr.header_pyramid(lib, ps, nplates)[3] == tr.pyramid_layout(ps, nplates)[2]
    if ps == 97:
        assert sizes == [97, 49, 25, 13, 7, 4, 2, 1]
    if ps == 2048:
        assert raw == 4 * 6 * sum(4 ** k for k in range(11)) and total == raw + 8   # (1024^2 + ... + 1) texels of 4 bytes on 6 plates
    if ps == 1:
        assert total == 0


def test_pyramid_beyond_fourteen_levels_is_refused(lib):
    assert tr.header_pyramid(lib, 8192, 6)[0] == 13   # 8192 halves to 1 in 13 steps
    assert tr.header_pyramid(lib, 8193, 6)[0] == -1 and tr.header_pyramid(lib, 1 << 14, 6)[0] == -1 and tr.header_pyramid(lib, 0, 6)[0] == -1


# ---- binding and host-only context -------------------------------------------------------------------------------

class FakeScratch(FakeCuda):
    """a contiguous CUDA tensor of n elements of `size` bytes at 1 MiB, for the binding"""

    def __init__(self, n, size=1):
        super().__init__((n,), "torch.uint8" if size == 1 else "torch.int32")
        self._size = size

    def numel(self):
        return self.shape[0]

    def element_size(self):
        return self._size

    def data_ptr(self):
        return 1 << 20

    def is_contiguous(self):
        return True


def panini(host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.command("f_fov 180")
    host.build_lensmap(W, H, PS, threads=1)


def test_binding_argument_checks(bb, host):
    panini(host)
    ok = FakeCuda((H, W, 3))
    for rays in (ok, FakeCuda((3, H, W, 3))):
        for scratch in (None, FakeScratch(1 << 20)):
            # past the checks, a host-only context refuses the call
            with pytest.raises(bb.BlinkyError) as e:
                host.warp_rays(0, 0, rays, FakeCuda((3, 3)), rgba=True, filter="trilinear", nframes=3, scratch=scratch)
            assert e.value.code == bb.E_NODEVICE
    with pytest.raises(ValueError, match="needs rgba=True"):
        host.warp_rays(0, 0, ok, filter="trilinear")
    for k in (2, 3, 4):
        with pytest.raises(ValueError, match="supersample=1"):
            host.warp_rays(0, 0, FakeCuda((k * H, k * W, 3)), rgba=True, supersample=k, filter="trilinear")
    with pytest.raises(ValueError, match="scratch is for filter='trilinear' only"):
        host.warp_rays(0, 0, ok, rgba=True, filter="bilinear", scratch=FakeScratch(16))
    with pytest.raises(ValueError, match=re.escape(f"rays must be float32 [{H}, {W}, 3]")):
        host.warp_rays(0, 0, FakeCuda((2 * H, 2 * W, 3)), rgba=True, filter="trilinear")
    for bad in ("Trilinear", "mip", None):
        with pytest.raises(ValueError, match="'trilinear'"):
            host.warp_rays(0, 0, ok, rgba=True, filter=bad)
    with pytest.raises(bb.BlinkyError) as e:
        host.ray_pyramid_bytes()
    assert e.value.code == bb.E_NODEVICE


def test_filter_selects_the_entry_point(bb, host, monkeypatch):
    """filter="trilinear" calls blinky_warp_device_rays_trilinear with the scratch's address and size"""
    panini(host)
    calls = []
    monkeypatch.setattr(host._lib, "blinky_warp_device_rays_trilinear", lambda *a: calls.append(a) or 0, raising=False)

    host.warp_rays(0, 0, FakeCuda((H, W, 3)), FakeCuda((2, 3, 3)), rgba=True, rowbytes=4 * W, screen_stride=4 * W * H, filter="trilinear",
                   keep_unmapped=True, scratch=FakeScratch(4096, 4))
    (a,) = calls
    assert a[12] == 2 and a[13] == 1 and a[16] == 1 << 20 and a[17] == 16384   # nframes, keep, d_scratch, scratch_bytes
    assert a[4] == 0 and a[6] == 36 and a[8] == 4 * W * H                       # ray_stride, xform_stride, screen stride


def test_host_only_context_refuses(bb, host):
    lib = bb.load_library()
    panini(host)
    rays = np.zeros((H, W, 3), np.float32)
    faces = np.zeros(6 * PS * PS, np.uint8)
    screen = np.zeros(4 * W * H, np.uint32)
    scratch = np.zeros(1 << 20, np.uint8)
    assert lib.blinky_warp_device_rays_trilinear(host._ctx, faces.ctypes.data, 0, rays.ctypes.data, 0, None, 0, screen.ctypes.data, 0, 4 * W, 0, 0,
                                                 1, 0, None, 0, scratch.ctypes.data, scratch.nbytes, None) == bb.E_NODEVICE
    n = ctypes.c_size_t(77)
    assert lib.blinky_ray_pyramid_bytes(host._ctx, ctypes.byref(n)) == bb.E_NODEVICE and n.value == 77
    assert host.launch_count == 0


# ---- the kernels' instances in the library ------------------------------------------------------------------------

INSTANCE = re.compile(r"ray_trilinear_kernelILb([01])ELb([01])ELb([01])EE")
WANT = {(r, kp, t) for r in (0, 1) for kp in (0, 1) for t in (0, 1)}
PYRAMID = re.compile(r"ray_pyramid_(base_kernelILb[01]ELb[01]EE|reduce_kernel)")


def test_the_trilinear_kernel_instances(bb):
    """<RUBIX, KEEP, TABLES>: 8 instances, each checked on the GPU by test_gpu_ray_trilinear.py::test_every_instance_follows_the_rule,
    and the pyramid kernels: 4 instances of the level-1 build (rubix, tables) and one reduction"""
    tool = shutil.which("cuobjdump") or next((p for p in ["/usr/local/cuda/bin/cuobjdump"] if os.path.exists(p)), None)
    if tool is None:
        pytest.skip("cuobjdump not found: cannot list the kernel instances of the built library")
    elf = subprocess.run([tool, "-elf", bb.LIB_PATH], check=True, capture_output=True, text=True).stdout
    names = {s for s in re.findall(r"\.text\.(\S+)", elf) if "ray_trilinear_kernel" in s}
    found = {tuple(int(b) for b in m.groups()) for s in names for m in [INSTANCE.search(s)] if m}
    assert len(names) == 8 and found == WANT, {"unexpected": sorted(found - WANT), "missing": sorted(WANT - found)}
    pyr = {m.group(1) for s in re.findall(r"\.text\.(\S+)", elf) for m in [PYRAMID.search(s)] if m}
    assert len(pyr) == 5, sorted(pyr)


def test_no_instance_spills(bb):
    """ptxas -v of csrc/ray_warp.cu (written by the build): no spill stores or loads in any trilinear or pyramid instance"""
    log = os.path.join(ROOT, "blinky_b200", "build", "ptxas_ray_warp.log")
    assert os.path.exists(log), "the build writes blinky_b200/build/ptxas_ray_warp.log"
    seen, pyr = set(), 0
    for chunk in open(log).read().split("Compiling entry function")[1:]:
        head = chunk.split("\n", 1)[0]
        m = INSTANCE.search(head)
        if not m and not PYRAMID.search(head):
            continue
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", chunk)
        assert spill and spill.groups() == ("0", "0"), (head, chunk[:400])
        if m:
            seen.add(tuple(int(b) for b in m.groups()))
        else:
            pyr += 1
    assert seen == WANT and pyr == 5, (sorted(WANT - seen), pyr)
