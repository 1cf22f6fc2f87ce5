"""The warp from a ray field turned by a per-frame matrix (blinky_warp_device_rays) without a GPU: the per-ray header
(ray_texel.h, compiled here with g++ -ffp-contract=off, as the kernel's translation unit is with --fmad=false) against
blinky_set_raymap of the field turned in numpy float32, entry for entry; the quad / pixel launch decision; the binding's
argument checks; the refusal of a host-only context; and the kernel's instances in the built library.  The GPU path is
tests/test_gpu_ray_warp.py."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_device_emulation import GRID
from test_globe_plate_transpile import params6
from test_raymap_host_only import adversarial_rays
from test_transpile import TRANSLATABLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, PS = 96, 64, 40
ARGMAX_GLOBES = ["cube", "cube_corner", "cube_edge", "tetra", "trism"]

SHIM = r"""
#include "ray_texel.h"
#include "launch_plan.h"
using namespace blinky;
extern "C" void entries(const LensBuildParams *P, const float *M, const float *rays, size_t n, uint32_t *out) {
    for (size_t i = 0; i < n; ++i) out[i] = ray_entry(*P, M, rays + 3 * i);
}
extern "C" int quads(int width, size_t opx, uintptr_t out, size_t pitch, size_t out_stride, int nframes) {
    WarpRequest r(nullptr, 0, reinterpret_cast<void *>(out), out_stride, nframes, nullptr);
    r.rgba = opx == 4;
    return ray_warp_quads(r, pitch, width);
}
extern "C" int frames_per_thread(size_t ray_stride, int nframes, uint32_t nitems, uint32_t resident) {
    return ray_warp_frames_per_thread(ray_stride, nframes, nitems, resident);
}
extern "C" void shape(int filter, int factor, int width, int height, int rgba, uintptr_t out, size_t pitch, size_t out_stride, int nframes,
                      size_t ray_stride, uint32_t resident, uint32_t *o) {
    WarpRequest r(nullptr, 0, reinterpret_cast<void *>(out), out_stride, nframes, nullptr);
    r.rgba = rgba != 0;
    RayRequest q = {nullptr, ray_stride, nullptr, 0};
    q.factor = factor;
    q.filter = static_cast<RayFilter>(filter);
    const RayWarpShape s = ray_warp_shape(r, q, pitch, width, height, resident);
    const uint32_t v[5] = {s.quads, s.nitems, static_cast<uint32_t>(s.frames_per_thread), s.grid_x, s.grid_y};
    for (int i = 0; i < 5; ++i) o[i] = v[i];
}
extern "C" const char *kernel_name(int filter, int factor) { return ray_warp_kernel_name(static_cast<RayFilter>(filter), factor); }
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("ray_texel")
    src = d / "shim.cpp"
    src.write_text(SHIM)
    so = d / "shim.so"
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-Wall", "-Wextra", "-shared", "-fPIC", "-I",
                        os.path.join(ROOT, "blinky_b200", "csrc"), "-o", str(so), str(src)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:3000]
    so_lib = ctypes.CDLL(str(so))
    so_lib.entries.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    so_lib.quads.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int]
    so_lib.frames_per_thread.argtypes = [ctypes.c_size_t, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32]
    so_lib.shape.argtypes = [ctypes.c_int] * 5 + [ctypes.c_size_t] * 3 + [ctypes.c_int, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_void_p]
    so_lib.kernel_name.argtypes = [ctypes.c_int, ctypes.c_int]
    so_lib.kernel_name.restype = ctypes.c_char_p
    return so_lib


def turned(rays, M):
    """numpy's float32 (M[k,0]*x + M[k,1]*y) + M[k,2]*z"""
    M = np.asarray(M, np.float32)
    x, y, z = rays[..., 0], rays[..., 1], rays[..., 2]
    with np.errstate(all="ignore"):
        return np.stack([(M[k, 0] * x + M[k, 1] * y) + M[k, 2] * z for k in range(3)], axis=-1).astype(np.float32)


def matrices(seed=0):
    """yaws, roll plus pitch, non-orthogonal, the identity; None is no turn"""
    rng = np.random.default_rng(seed)
    out = []
    for deg in (0.0, 37.0, 90.0, -135.0, 180.0):
        a = np.radians(deg)
        out.append(np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32))
    a, b = np.radians(12.0), np.radians(-48.0)
    roll = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], np.float32)
    pitch = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]], np.float32)
    out.append((roll @ pitch).astype(np.float32))
    out.append((np.eye(3) + 0.4 * rng.normal(size=(3, 3))).astype(np.float32))
    out.append(rng.normal(size=(3, 3)).astype(np.float32) * np.float32(1e19))   # overflowing products
    out.append(np.eye(3, dtype=np.float32))
    return out + [None]


def params(host, w, h, ps, grid):
    slots = np.zeros((6, 11), np.float32)
    pl = host.plates()
    slots[: len(pl)] = pl
    p = params6(host, w, h, ps, slots)
    numcells, cell, pad = grid
    p.rubix_block = pad + cell
    p.rubix_pad = pad
    p.rubix_unit_px = float(ps) / (numcells * p.rubix_block + pad)
    return p


def header_entries(lib, p, M, rays):
    flat = np.ascontiguousarray(rays.reshape(-1, 3), np.float32)
    out = np.zeros(len(flat), np.uint32)
    m = None if M is None else np.ascontiguousarray(M, np.float32)
    lib.entries(ctypes.byref(p), None if m is None else m.ctypes.data, flat.ctypes.data, len(flat), out.ctypes.data)
    return out


def assert_header_equals_set_raymap(lib, host, rays, M, ps, grid, what):
    h, w = rays.shape[:2]
    t = rays if M is None else turned(rays, M)
    with np.errstate(all="ignore"):
        host.set_raymap(np.ascontiguousarray(t), ps)
    want = host.lensmap_packed().reshape(-1)
    got = header_entries(lib, params(host, w, h, ps, grid), M, rays)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, (what, bad.size, [(rays.reshape(-1, 3)[i].tolist(), hex(got[i]), hex(want[i])) for i in bad[:4]])
    return want


def test_every_translatable_lens_turned(lib, host):
    host.command("f_globe cube")
    host.set_rubixgrid(*GRID)
    checked = 0
    for lens in TRANSLATABLE:
        host.command(f"f_lens {lens}")
        host.command("f_fov 180")
        try:
            rays = host.raymap(W, H)
        except Exception:  # noqa: BLE001 — a zoom this lens cannot do
            continue
        for i, M in enumerate(matrices()):
            assert_header_equals_set_raymap(lib, host, rays, M, PS, GRID, (lens, i))
        checked += 1
    assert checked >= 15, checked


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
    mapped = 0
    for i, M in enumerate(matrices(seed=len(globe))):
        want = assert_header_equals_set_raymap(lib, host, rays, M, 37, grid, (globe, i))
        mapped += int(((want >> 31) & 1).sum())
        if i == 0:
            tints = (want >> 28) & 7
            assert (tints[(want >> 31) == 1] == 7).any(), "some texels on the rubix grid"
    assert mapped > 0


@pytest.mark.parametrize("globe", ARGMAX_GLOBES)
def test_adversarial_rays(lib, host, globe):
    """zeros, -0, NaN, +-inf, subnormals, +-3e38, rays on plate edges and corners (u or v exactly 0 or 1, u * ps
    reaching ps) and cube-corner ties, turned by every matrix and not at all"""
    host.set_rubixgrid(*GRID)
    host.command(f"f_globe {globe}")
    slots = np.zeros((6, 11), np.float32)
    pl = host.plates()
    slots[: len(pl)] = pl
    ps = 64
    rays = adversarial_rays(slots, len(pl), ps)
    extra = np.array([[-3e38, 3e38, 1], [-0.0, -0.0, 1], [1, -0.0, 0], [np.float32(1e-45), 1, 0], [1, 1, np.nan]], np.float32)
    rays = np.vstack([rays, extra])
    n = len(rays)
    w = 50
    h = -(-n // w)
    field = np.zeros((h * w, 3), np.float32)
    field[:n] = rays
    field = field.reshape(h, w, 3)
    for i, M in enumerate(matrices(seed=3)):
        assert_header_equals_set_raymap(lib, host, field, M, ps, GRID, (globe, i))


# ---- launch decision ---------------------------------------------------------------------------------------------

def test_launch_decision(lib):
    q = lib.quads
    # 8-bit: 4-byte words; RGBA: 16-byte words
    assert q(96, 1, 4096, 128, 8192, 3) == 1
    assert q(96, 1, 4096 + 3, 128, 8192, 3) == 0, "odd view origin"
    assert q(96, 1, 4096, 127, 8192, 3) == 0, "odd pitch"
    assert q(96, 1, 4096, 128, 8190, 3) == 0, "odd frame stride"
    assert q(96, 1, 4096, 128, 8190, 1) == 1, "one frame: the stride is never used"
    assert q(94, 1, 4096, 128, 8192, 3) == 0, "W % 4 != 0: a quad would straddle two rows"
    assert q(96, 4, 4096 + 4, 512, 65536, 2) == 0 and q(96, 4, 4096 + 16, 512, 65536, 2) == 1
    assert q(96, 4, 4096, 392, 65536, 2) == 0 and q(96, 4, 4096, 400, 65536, 2) == 1
    fpt = lib.frames_per_thread
    resident = 132 * 2048
    # 4K quads fill the GPU alone: every frame in one thread, the field read once per launch
    assert fpt(0, 16, 3840 * 2160 // 4, resident) == 16 and fpt(0, 60, 3840 * 2160 // 4, resident) == 60
    assert fpt(0, 1, 3840 * 2160 // 4, resident) == 1
    # per-frame fields: one frame per thread
    assert fpt(12 * 96 * 64, 16, 96 * 64 // 4, resident) == 1 and fpt(12 * 3840 * 2160, 16, 3840 * 2160 // 4, resident) == 1
    # a small view: the frames are split until the launch holds a GPU's worth of threads
    assert fpt(0, 5, 1536, resident) == 1
    assert fpt(0, 400, 1536, resident) == 2      # 176 rows of threads wanted, 200 launched
    assert fpt(0, 65535, 1536, resident) == 372
    for nitems in (1, 7, 1536, 100000, 270336, 270337, 2073600):
        for n in (1, 2, 3, 17, 176, 177, 1000, 65535):
            f = fpt(0, n, nitems, resident)
            rows = -(-n // f)
            assert 1 <= f <= n
            assert rows * nitems >= min(resident, n * nitems), (nitems, n, f)   # enough threads, when there are enough frames
            assert f == 1 or (rows - 1) * nitems < 2 * resident, (nitems, n, f)   # and not many more


NEAREST, BILINEAR, TRILINEAR = 0, 1, 2   # RayFilter


def test_launch_shape(lib):
    """ray_warp_shape over every filter and factor, on aligned and unaligned views: quads only for the nearest filter at
    factor 1 (a quad instance launched with one item per pixel would read rays and background four times past their
    end), and a grid that covers every item and every frame"""
    o = np.zeros(5, np.uint32)
    resident = 132 * 2048
    seen = set()
    for filt, factors in ((NEAREST, (1, 2, 3, 4)), (BILINEAR, (1, 2, 3, 4)), (TRILINEAR, (1,))):
        for k in factors:
            for w, h in ((96, 64), (94, 64), (3840, 2160), (640, 480), (1, 1), (5, 3), (4, 1)):
                for rgba in ((0, 1) if filt == NEAREST and k == 1 else (1,)):
                    opx = 4 if rgba else 1
                    pitch = -(-w * opx // 16) * 16
                    for origin, p in ((4096, pitch), (4096 + opx, pitch), (4096, pitch + opx)):
                        for ray_stride in (0, 12 * k * k * w * h):
                            for n in (1, 3, 400):
                                lib.shape(filt, k, w, h, rgba, origin, p, p * h, n, ray_stride, resident, o.ctypes.data)
                                quads, nitems, fpt, gx, gy = (int(v) for v in o)
                                what = (filt, k, w, h, rgba, origin, p, ray_stride, n, o.tolist())
                                if quads:
                                    assert filt == NEAREST and k == 1 and w % 4 == 0 and nitems * 4 == w * h, what
                                else:
                                    assert nitems == w * h, what
                                assert gx * 256 >= nitems > (gx - 1) * 256, what
                                assert 1 <= fpt <= n and gy * fpt >= n > (gy - 1) * fpt, what
                                assert fpt == 1 or ray_stride == 0, what
                                seen.add((filt, k, quads))
    assert (NEAREST, 1, 1) in seen and (NEAREST, 1, 0) in seen
    assert lib.kernel_name(NEAREST, 1) == b"ray_warp_kernel"
    assert all(lib.kernel_name(NEAREST, k) == b"ray_supersample_kernel" for k in (2, 3, 4))
    assert all(lib.kernel_name(BILINEAR, k) == b"ray_bilinear_kernel" for k in (1, 2, 3, 4))
    assert lib.kernel_name(TRILINEAR, 1) == b"ray_trilinear_kernel"


# ---- binding and host-only context -------------------------------------------------------------------------------

class FakeCuda:
    """just enough of a CUDA tensor for the binding's checks, which run before any call"""

    def __init__(self, shape, dtype="torch.float32", strides=None):
        self.shape = tuple(shape)
        self.dtype = dtype
        self.is_cuda = True
        st, acc = [], 1
        for s in reversed(self.shape):
            st.append(acc)
            acc *= s
        self._strides = tuple(strides) if strides else tuple(reversed(st))

    def dim(self):
        return len(self.shape)

    def stride(self, i=None):
        return self._strides if i is None else self._strides[i]

    def data_ptr(self):
        return 0


def test_binding_argument_checks(bb, host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.command("f_fov 180")
    host.build_lensmap(W, H, PS, threads=1)
    ok_rays = FakeCuda((H, W, 3))
    with pytest.raises(TypeError, match="CUDA tensor"):
        host.warp_rays(0, 0, np.zeros((H, W, 3), np.float32))
    cases = [FakeCuda((H, W, 3), dtype="torch.float64"), FakeCuda((H, W - 1, 3)), FakeCuda((W, H, 3)), FakeCuda((2, 2, H, W, 3)),
             FakeCuda((H, W, 3), strides=(3 * W + 3, 3, 1)), FakeCuda((H, W, 4))]
    for r in cases:
        with pytest.raises(ValueError, match="rays must be"):
            host.warp_rays(0, 0, r)
    with pytest.raises(TypeError, match="xforms must be a CUDA tensor"):
        host.warp_rays(0, 0, ok_rays, np.eye(3, dtype=np.float32))
    for x in [FakeCuda((3, 3), dtype="torch.float16"), FakeCuda((3, 4)), FakeCuda((2, 3, 3), strides=(9, 1, 3)), FakeCuda((9,))]:
        with pytest.raises(ValueError, match="xforms must be"):
            host.warp_rays(0, 0, ok_rays, x)
    with pytest.raises(ValueError, match="2 ray fields for 3 frames"):
        host.warp_rays(0, 0, FakeCuda((2, H, W, 3)), nframes=3)
    with pytest.raises(ValueError, match="2 matrices for 3 frames"):
        host.warp_rays(0, 0, ok_rays, FakeCuda((2, 3, 3)), nframes=3)
    with pytest.raises(ValueError, match="rgba"):
        host.warp_rays(0, 0, ok_rays, tables=FakeCuda((256,)))
    # past the checks, a host-only context refuses the call
    with pytest.raises(bb.BlinkyError) as e:
        host.warp_rays(0, 0, FakeCuda((3, H, W, 3)), FakeCuda((3, 3, 3)))
    assert e.value.code == bb.E_NODEVICE


def test_host_only_context_refuses(bb, host):
    lib = bb.load_library()
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.build_lensmap(W, H, PS, threads=1)
    rays = np.zeros((H, W, 3), np.float32)
    faces = np.zeros(6 * PS * PS, np.uint8)
    screen = np.zeros(4 * W * H, np.uint8)
    m = np.eye(3, dtype=np.float32)
    before = host.launch_count
    assert lib.blinky_warp_device_rays(host._ctx, faces.ctypes.data, 0, rays.ctypes.data, 0, m.ctypes.data, 0, screen.ctypes.data, 0, W, 0, 0, 1, 0,
                                       None) == bb.E_NODEVICE
    assert lib.blinky_warp_device_rays_rgba(host._ctx, faces.ctypes.data, 0, rays.ctypes.data, 0, None, 0, screen.ctypes.data, 0, 4 * W, 0, 0, 1,
                                            0, None, 0, None) == bb.E_NODEVICE
    assert host.launch_count == before == 0


# ---- the kernel's instances in the library -----------------------------------------------------------------------

RAY_INSTANCE = re.compile(r"ray_warp_kernelILb([01])ELb([01])ELb([01])ELb([01])ELb([01])EE")


def test_the_ray_warp_kernel_instances(bb):
    """<QUAD, RUBIX, RGBA, KEEP, TABLES>: every combination with per-frame tables only in RGBA — 24 instances, each
    checked on the GPU by test_gpu_ray_warp.py::test_every_instance_follows_the_rule"""
    tool = shutil.which("cuobjdump") or next((p for p in ["/usr/local/cuda/bin/cuobjdump"] if os.path.exists(p)), None)
    if tool is None:
        pytest.skip("cuobjdump not found: cannot list the kernel instances of the built library")
    elf = subprocess.run([tool, "-elf", bb.LIB_PATH], check=True, capture_output=True, text=True).stdout
    found = {tuple(int(b) for b in m.groups()) for s in re.findall(r"\.text\.(\S+)", elf) for m in [RAY_INSTANCE.search(s)] if m}
    want = {(q, r, c, k, t) for q in (0, 1) for r in (0, 1) for c in (0, 1) for k in (0, 1) for t in (0, 1) if c or not t}
    assert len(want) == 24
    assert found == want, {"unexpected": sorted(found - want), "missing": sorted(want - found)}
