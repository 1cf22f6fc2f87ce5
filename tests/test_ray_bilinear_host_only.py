"""The bilinear warp from a ray field (blinky_warp_device_rays_bilinear, Fisheye.warp_rays(filter="bilinear")) without
a GPU: the per-ray header function ray_bilinear and the per-axis grid test ray_on_rubix_line (ray_texel.h, compiled with
g++ -ffp-contract=off behind tests/ray_bilinear_reference.py's shim, as the kernel's translation unit is with --fmad=false) against ray_entry and an independent
numpy restatement of the rule; the binding's argument checks; the refusal of a host-only context; and the kernel's
instances in the built library and in its ptxas log.  The GPU path is tests/test_gpu_ray_bilinear.py."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from ray_bilinear_reference import compile_shim, header_samples
from test_device_emulation import GRID
from test_ray_warp_host_only import ARGMAX_GLOBES, FakeCuda, matrices, params, turned
from test_raymap_host_only import adversarial_rays
from test_transpile import TRANSLATABLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, PS = 96, 64, 40

@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return compile_shim(tmp_path_factory.mktemp("ray_bilinear"))


def restated(p, rays):
    """the rule in numpy, from the turned rays [n, 3]: (mapped, plate, x0, y0, wx, wy).  The ray is normalised and dotted
    in float32 (each product and sum rounded, left to right), the plate is the strict argmax of the widened dots
    (lowest index on ties, NaN never wins), u and v are float64, and the sample is mapped when u, v lie in [0, 1] and
    their texels (int)(u ps), (int)(v ps) lie below ps.  Then sx = u ps - 0.5, x0 = floor(sx), wx = (int)((sx - x0) 256)."""
    r = np.ascontiguousarray(rays, np.float32).copy()
    n = len(r)
    f32 = np.float32
    with np.errstate(all="ignore"):
        ln = (r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2]
        ln = np.sqrt(ln.astype(np.float64)).astype(f32)
        inv = f32(1) / ln
        r = np.where((ln != 0)[:, None], r * inv[:, None], r)

        def dot(vec):
            a = np.asarray(vec, f32)
            return ((r[:, 0] * a[0] + r[:, 1] * a[1]) + r[:, 2] * a[2]).astype(np.float64)

        best = np.zeros(n, np.int64)
        best_dp = np.full(n, -2.0)
        for i in range(p.numplates):
            dp = dot(p.plates[i].forward)
            win = dp > best_dp
            best = np.where(win, i, best)
            best_dp = np.where(win, dp, best_dp)
        x, y, z = (np.zeros(n) for _ in range(3))
        uvd = np.zeros(n)
        for i in range(p.numplates):
            sel = best == i
            pl = p.plates[i]
            x[sel], y[sel], z[sel] = dot(pl.right)[sel], dot(pl.up)[sel], dot(pl.forward)[sel]
            uvd[sel] = p.uv_dist[i]
        u = x / z * uvd + 0.5
        v = -y / z * uvd + 0.5
        ps = p.platesize
        ok = (u >= 0) & (u <= 1) & (v >= 0) & (v <= 1)
        uu, vv = np.where(ok, u, 0.0), np.where(ok, v, 0.0)
        mapped = ok & (np.trunc(uu * ps) < ps) & (np.trunc(vv * ps) < ps)
        sx, sy = uu * ps - 0.5, vv * ps - 0.5
        x0, y0 = np.floor(sx), np.floor(sy)
        wx, wy = np.trunc((sx - x0) * 256), np.trunc((sy - y0) * 256)
    return mapped, best, x0.astype(np.int64), y0.astype(np.int64), wx.astype(np.int64), wy.astype(np.int64)


def assert_follows_the_rule(lib, p, rays, M, what):
    """ray_bilinear against ray_entry (mapped-ness and plate) and the restatement (positions); the mapped samples'
    (x0, y0, wx, wy)"""
    entry, got = header_samples(lib, p, M, rays)
    flat = rays.reshape(-1, 3)
    t = flat if M is None else turned(flat, M)
    mapped, plate, x0, y0, wx, wy = restated(p, t)
    ps = p.platesize
    e_mapped = (entry >> 31) == 1
    e_plate = (entry & 0x0FFFFFFF).astype(np.int64) // (ps * ps)
    m = got[:, 0] == 1
    bad = np.nonzero((m != e_mapped) | (m & (got[:, 1] != e_plate)))[0]
    assert bad.size == 0, (what, "ray_entry", bad.size, [(flat[i].tolist(), hex(entry[i]), got[i].tolist()) for i in bad[:4]])
    bad = np.nonzero(m != mapped)[0]
    assert bad.size == 0, (what, "mapped", bad.size, [(flat[i].tolist(), got[i].tolist()) for i in bad[:4]])
    want = np.stack([plate, x0, y0, wx, wy], axis=1)[m]
    bad = np.nonzero((got[m, 1:] != want).any(axis=1))[0]
    assert bad.size == 0, (what, "positions", bad.size, [(got[m][i].tolist(), want[i].tolist()) for i in bad[:4]])
    s = got[m]
    assert (s[:, 2:4] >= -1).all() and (s[:, 2:4] <= ps - 1).all() and (s[:, 4:6] >= 0).all() and (s[:, 4:6] <= 255).all(), what
    return s


def test_every_translatable_lens_turned(lib, host):
    host.command("f_globe cube")
    host.set_rubixgrid(*GRID)
    checked = 0
    weights = set()
    for lens in TRANSLATABLE:
        host.command(f"f_lens {lens}")
        host.command("f_fov 180")
        try:
            rays = host.raymap(W, H)
        except Exception:  # noqa: BLE001 — a zoom this lens cannot do
            continue
        p = params(host, W, H, PS, GRID)
        for i, M in enumerate(matrices()):
            s = assert_follows_the_rule(lib, p, rays, M, (lens, i))
            weights.update(s[:, 4].tolist())
        checked += 1
    assert checked >= 15, checked
    assert len(weights) > 200, "the weights cover their range"


@pytest.mark.parametrize("grid", [GRID, (4, 3.0, 2.0)])
@pytest.mark.parametrize("globe", ARGMAX_GLOBES)
def test_argmax_globes_and_grids(lib, host, globe, grid):
    host.set_rubixgrid(*grid)
    host.command(f"f_globe {globe}")
    host.command("f_lens panini")
    host.command("f_fov 180")
    rays = host.raymap(W, H)
    rng = np.random.default_rng(len(globe))
    rays.reshape(-1, 3)[::7] = rng.normal(size=rays.reshape(-1, 3)[::7].shape).astype(np.float32)
    ps = 37
    p = params(host, W, H, ps, grid)
    mapped = 0
    for i, M in enumerate(matrices(seed=len(globe))):
        mapped += len(assert_follows_the_rule(lib, p, rays, M, (globe, i)))
    assert mapped > 0
    # the per-axis test: a texel is on the grid exactly when its column or its row is
    line = np.zeros(ps, np.uint8)
    cell = np.zeros(ps * ps, np.uint8)
    lib.grid(ctypes.byref(p), ps, line.ctypes.data, cell.ctypes.data)
    assert 0 < line.sum() < ps
    assert np.array_equal(cell.reshape(ps, ps).astype(bool), line.astype(bool)[None, :] | line.astype(bool)[:, None]), (globe, grid)


@pytest.mark.parametrize("globe", ARGMAX_GLOBES)
def test_adversarial_rays(lib, host, globe):
    """zeros, -0, NaN, +-inf, subnormals, +-3e38, rays on plate edges and corners (u or v exactly 0 or 1, u * ps
    reaching ps) and cube-corner ties, turned by every matrix and not at all.  On the cube globes, whose plates meet at
    their edges, the taps' first coordinate reaches both -1 (u * ps < 0.5) and ps - 1."""
    host.set_rubixgrid(*GRID)
    host.command(f"f_globe {globe}")
    slots = np.zeros((6, 11), np.float32)
    pl = host.plates()
    slots[: len(pl)] = pl
    ps = 64
    rays = adversarial_rays(slots, len(pl), ps)
    extra = np.array([[-3e38, 3e38, 1], [-0.0, -0.0, 1], [1, -0.0, 0], [np.float32(1e-45), 1, 0], [1, 1, np.nan]], np.float32)
    rays = np.vstack([rays, extra])
    p = params(host, 50, 50, ps, GRID)
    corners = set()
    for i, M in enumerate(matrices(seed=3)):
        s = assert_follows_the_rule(lib, p, rays, M, (globe, i))
        corners.update(s[:, 2].tolist())
        corners.update(s[:, 3].tolist())
    if globe.startswith("cube"):
        assert -1 in corners and ps - 1 in corners, sorted(corners)[:3]


# ---- binding and host-only context -------------------------------------------------------------------------------

def panini(host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.command("f_fov 180")
    host.build_lensmap(W, H, PS, threads=1)


def test_binding_argument_checks(bb, host):
    panini(host)
    for k in (1, 2, 3, 4):
        ok = FakeCuda((k * H, k * W, 3))
        # past the checks, a host-only context refuses the call
        for rays in (ok, FakeCuda((3, k * H, k * W, 3))):
            with pytest.raises(bb.BlinkyError) as e:
                host.warp_rays(0, 0, rays, FakeCuda((3, 3)), rgba=True, supersample=k, filter="bilinear", nframes=3)
            assert e.value.code == bb.E_NODEVICE
        for rays in (FakeCuda((k * H + 1, k * W, 3)), FakeCuda((k * H, k * W, 3), strides=(3 * k * W + 3, 3, 1)),
                     FakeCuda((k * H, k * W, 3), dtype="torch.float64")):
            with pytest.raises(ValueError, match=re.escape(f"rays must be float32 [{k * H}, {k * W}, 3] or [N, {k * H}, {k * W}, 3]")):
                host.warp_rays(0, 0, rays, rgba=True, supersample=k, filter="bilinear")
        # palette indices cannot be blended
        with pytest.raises(ValueError, match="needs rgba=True"):
            host.warp_rays(0, 0, ok, supersample=k, filter="bilinear")
    for bad in ("linear", "Bilinear", "", None, 1):
        with pytest.raises(ValueError, match="filter must be 'nearest' or 'bilinear'"):
            host.warp_rays(0, 0, FakeCuda((H, W, 3)), rgba=True, filter=bad)
    for bad in (0, 5):
        with pytest.raises(ValueError, match="supersample must be 1, 2, 3 or 4"):
            host.warp_rays(0, 0, FakeCuda((H, W, 3)), rgba=True, supersample=bad, filter="bilinear")


def test_filter_selects_the_entry_point(bb, host, monkeypatch):
    """filter="nearest" is a call without it; "bilinear" calls blinky_warp_device_rays_bilinear with the factor"""
    panini(host)
    calls = []
    for name in ("blinky_warp_device_rays", "blinky_warp_device_rays_rgba", "blinky_warp_device_rays_supersampled",
                 "blinky_warp_device_rays_bilinear"):
        monkeypatch.setattr(host._lib, name, lambda *a, _n=name: calls.append((_n, a)) or 0, raising=False)
    for k, name in ((1, "blinky_warp_device_rays_rgba"), (2, "blinky_warp_device_rays_supersampled")):
        calls.clear()
        rays = FakeCuda((k * H, k * W, 3))
        host.warp_rays(0, 0, rays, rgba=True, rowbytes=4 * W, screen_stride=4 * W * H, supersample=k)
        host.warp_rays(0, 0, rays, rgba=True, rowbytes=4 * W, screen_stride=4 * W * H, supersample=k, filter="nearest")
        assert [c[0] for c in calls] == [name] * 2 and calls[0][1] == calls[1][1]
    for k in (1, 2, 3, 4):
        calls.clear()
        host.warp_rays(0, 0, FakeCuda((k * H, k * W, 3)), rgba=True, rowbytes=4 * W, screen_stride=4 * W * H, supersample=k, filter="bilinear",
                       nframes=2, keep_unmapped=True)
        (name, a), = calls
        assert name == "blinky_warp_device_rays_bilinear"
        assert a[7] == k and a[4] == 0 and a[9] == 4 * W * H and a[13] == 2 and a[14] == 1   # factor, ray_stride, screen stride, nframes, keep


def test_host_only_context_refuses(bb, host):
    lib = bb.load_library()
    panini(host)
    rays = np.zeros((2 * H, 2 * W, 3), np.float32)
    faces = np.zeros(6 * PS * PS, np.uint8)
    screen = np.zeros(4 * W * H, np.uint32)
    for factor in (0, 1, 2, 5):
        assert lib.blinky_warp_device_rays_bilinear(host._ctx, faces.ctypes.data, 0, rays.ctypes.data, 0, None, 0, factor, screen.ctypes.data, 0,
                                                    4 * W, 0, 0, 1, 0, None, 0, None) == bb.E_NODEVICE
    assert host.launch_count == 0


# ---- the kernel's instances in the library -----------------------------------------------------------------------

INSTANCE = re.compile(r"ray_bilinear_kernelILi([1234])ELb([01])ELb([01])ELb([01])EE")
WANT = {(k, r, kp, t) for k in (1, 2, 3, 4) for r in (0, 1) for kp in (0, 1) for t in (0, 1)}


def test_the_bilinear_kernel_instances(bb):
    """<K, RUBIX, KEEP, TABLES>: 4 x 2 x 2 x 2 = 32 instances, each checked on the GPU by
    test_gpu_ray_bilinear.py::test_every_instance_follows_the_rule"""
    tool = shutil.which("cuobjdump") or next((p for p in ["/usr/local/cuda/bin/cuobjdump"] if os.path.exists(p)), None)
    if tool is None:
        pytest.skip("cuobjdump not found: cannot list the kernel instances of the built library")
    elf = subprocess.run([tool, "-elf", bb.LIB_PATH], check=True, capture_output=True, text=True).stdout
    names = {s for s in re.findall(r"\.text\.(\S+)", elf) if "ray_bilinear_kernel" in s}
    found = {tuple(int(b) for b in m.groups()) for s in names for m in [INSTANCE.search(s)] if m}
    assert len(WANT) == 32
    assert len(names) == 32 and found == WANT, {"unexpected": sorted(found - WANT), "missing": sorted(WANT - found), "names": len(names)}


def test_no_instance_spills(bb):
    """ptxas -v of csrc/ray_warp.cu (written by the build): no spill stores or loads in any bilinear instance"""
    log = os.path.join(ROOT, "blinky_b200", "build", "ptxas_ray_warp.log")
    assert os.path.exists(log), "the build writes blinky_b200/build/ptxas_ray_warp.log"
    text = open(log).read()
    seen = set()
    for chunk in text.split("Compiling entry function")[1:]:
        m = INSTANCE.search(chunk.split("\n", 1)[0])
        if not m:
            continue
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", chunk)
        assert spill, chunk[:400]
        assert spill.groups() == ("0", "0"), (m.group(0), spill.group(0))
        seen.add(tuple(int(b) for b in m.groups()))
    assert seen == WANT, sorted(WANT - seen)
