"""The supersampled warp from a ray field (blinky_warp_device_rays_supersampled, Fisheye.warp_rays(supersample=k))
without a GPU: the binding's argument checks, the refusal of a host-only context, and the kernel's instances in the
built library and in its ptxas log.  The GPU path is tests/test_gpu_ray_supersample.py."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_ray_warp_host_only import FakeCuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, PS = 96, 64, 40


def panini(host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.command("f_fov 180")
    host.build_lensmap(W, H, PS, threads=1)


def test_binding_argument_checks(bb, host):
    panini(host)
    for k in (2, 3, 4):
        ok = FakeCuda((k * H, k * W, 3))
        # past the checks, a host-only context refuses the call
        for rays in (ok, FakeCuda((3, k * H, k * W, 3))):
            with pytest.raises(bb.BlinkyError) as e:
                host.warp_rays(0, 0, rays, FakeCuda((3, 3)), rgba=True, supersample=k, nframes=3)
            assert e.value.code == bb.E_NODEVICE
        # the field must be the k-fold one, and the message names it
        for rays in (FakeCuda((H, W, 3)), FakeCuda((k * H, k * W - 1, 3)), FakeCuda((k * W, k * H, 3)),
                     FakeCuda((k * H, k * W, 3), strides=(3 * k * W + 3, 3, 1)), FakeCuda((k * H, k * W, 3), dtype="torch.float64"),
                     FakeCuda((2, 2, k * H, k * W, 3))):
            with pytest.raises(ValueError, match=re.escape(f"rays must be float32 [{k * H}, {k * W}, 3] or [N, {k * H}, {k * W}, 3]")):
                host.warp_rays(0, 0, rays, rgba=True, supersample=k)
        with pytest.raises(ValueError, match="2 ray fields for 3 frames"):
            host.warp_rays(0, 0, FakeCuda((2, k * H, k * W, 3)), rgba=True, supersample=k, nframes=3)
        # palette indices cannot be averaged
        with pytest.raises(ValueError, match="rgba=True"):
            host.warp_rays(0, 0, ok, supersample=k)
    # a k-fold field is not a one-sample field
    with pytest.raises(ValueError, match=re.escape(f"rays must be float32 [{H}, {W}, 3]")):
        host.warp_rays(0, 0, FakeCuda((2 * H, 2 * W, 3)), rgba=True)
    for bad in (0, 5, -1):
        with pytest.raises(ValueError, match="supersample must be 1, 2, 3 or 4"):
            host.warp_rays(0, 0, FakeCuda((H, W, 3)), rgba=True, supersample=bad)
    for bad in (2.0, "2", True, None):
        with pytest.raises(TypeError, match="supersample must be an int"):
            host.warp_rays(0, 0, FakeCuda((H, W, 3)), rgba=True, supersample=bad)


def test_supersample_one_is_the_one_sample_call(bb, host, monkeypatch):
    """supersample=1 takes blinky_warp_device_rays[_rgba] with the arguments of a call without it"""
    panini(host)
    calls = []
    for name in ("blinky_warp_device_rays", "blinky_warp_device_rays_rgba", "blinky_warp_device_rays_supersampled"):
        monkeypatch.setattr(host._lib, name, lambda *a, _n=name: calls.append((_n, a)) or 0, raising=False)
    rays = FakeCuda((H, W, 3))
    for rgba in (False, True):
        calls.clear()
        host.warp_rays(0, 0, rays, rgba=rgba, rowbytes=4 * W, screen_stride=4 * W * H)
        host.warp_rays(0, 0, rays, rgba=rgba, rowbytes=4 * W, screen_stride=4 * W * H, supersample=1)
        assert [c[0] for c in calls] == ["blinky_warp_device_rays_rgba" if rgba else "blinky_warp_device_rays"] * 2
        assert calls[0][1] == calls[1][1]
    calls.clear()
    host.warp_rays(0, 0, FakeCuda((3 * H, 3 * W, 3)), rgba=True, rowbytes=4 * W, screen_stride=4 * W * H, supersample=3, nframes=2)
    (name, a), = calls
    assert name == "blinky_warp_device_rays_supersampled"
    assert a[7] == 3 and a[4] == 0 and a[9] == 4 * W * H and a[13] == 2   # factor, ray_stride, screen stride, nframes


def test_host_only_context_refuses(bb, host):
    lib = bb.load_library()
    panini(host)
    rays = np.zeros((2 * H, 2 * W, 3), np.float32)
    faces = np.zeros(6 * PS * PS, np.uint8)
    screen = np.zeros(4 * W * H, np.uint32)
    for factor in (1, 2, 5):
        assert lib.blinky_warp_device_rays_supersampled(host._ctx, faces.ctypes.data, 0, rays.ctypes.data, 0, None, 0, factor, screen.ctypes.data, 0,
                                                        4 * W, 0, 0, 1, 0, None, 0, None) == bb.E_NODEVICE
    assert host.launch_count == 0


# ---- the kernel's instances in the library -----------------------------------------------------------------------

INSTANCE = re.compile(r"ray_supersample_kernelILi([234])ELb([01])ELb([01])ELb([01])EE")
WANT = {(k, r, kp, t) for k in (2, 3, 4) for r in (0, 1) for kp in (0, 1) for t in (0, 1)}


def test_the_supersample_kernel_instances(bb):
    """<K, RUBIX, KEEP, TABLES>: 3 x 2 x 2 x 2 = 24 instances, each checked on the GPU by
    test_gpu_ray_supersample.py::test_every_instance_follows_the_rule"""
    tool = shutil.which("cuobjdump") or next((p for p in ["/usr/local/cuda/bin/cuobjdump"] if os.path.exists(p)), None)
    if tool is None:
        pytest.skip("cuobjdump not found: cannot list the kernel instances of the built library")
    elf = subprocess.run([tool, "-elf", bb.LIB_PATH], check=True, capture_output=True, text=True).stdout
    names = {s for s in re.findall(r"\.text\.(\S+)", elf) if "ray_supersample_kernel" in s}
    found = {tuple(int(b) for b in m.groups()) for s in names for m in [INSTANCE.search(s)] if m}
    assert len(WANT) == 24
    assert len(names) == 24 and found == WANT, {"unexpected": sorted(found - WANT), "missing": sorted(WANT - found), "names": len(names)}


def test_no_instance_spills(bb):
    """ptxas -v of csrc/ray_warp.cu (written by the build): no spill stores or loads in any supersampled instance"""
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
