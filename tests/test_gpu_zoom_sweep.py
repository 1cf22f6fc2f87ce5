"""The GPU lens build (build_lensmap(threads=0)) and the GPU ray export (raymap into a CUDA tensor) against the interpreter
over the zoom and view-shape sweep of zoom_sweep.py: every shipped lens at every zoom of the sweep and every view shape
on cube, and the reduced sweep on the five other globes, rubix off and on (a non-default grid for half of the rubix
cases).  The interpreter's side runs on a second, host-only context, so the two paths share nothing but the scripts.

For each case: the same error code and log (the "> maxdiff" lines of the forward builder in order, the refusal message
of a zoom past a lens's limit), the same lensmap, display flags and scale, bit for bit; and for an inverse lens the same
exported rays.  Translatable lenses must take the device path and forward-only lenses the forward device path.  With -s
the share of pixels (grid points for forward lenses) the interpreter had to settle is printed for the cases where it is
above 1 %."""
import re
import time

import numpy as np
import pytest

from conftest import ALL_LENSES
from test_raymap_export_host_only import assert_same_rays
from test_transpile import FORWARD_ONLY, TRANSLATABLE
from zoom_sweep import REDUCED_GLOBES, SHAPES, reduced_cases, refused_past_the_limit, zoom_limits, zooms

pytestmark = pytest.mark.gpu

DEFAULT_GRID = (10, 4.0, 1.0)   # f_rubixgrid's default
OTHER_GRID = (4, 3.0, 2.0)


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture()
def pair(bb, palette, cuda_device):
    """(the GPU context, the host-only context that builds and exports with the interpreter)"""
    dev = bb.Fisheye(device=cuda_device, palette=palette)
    ref = bb.Fisheye(device=None, palette=palette)
    yield dev, ref
    dev.close()
    ref.close()


def build(bb, fe, w, h, ps, threads):
    fe.clear_log()
    try:
        fe.build_lensmap(w, h, ps, threads=threads)
        code = 0
    except bb.BlinkyError as e:
        code = e.code
    idx, tint = fe.lensmap()
    return code, idx, tint, fe.display(), fe.log, np.float64(fe.scale).tobytes()


def undecided_share(info):
    """(undecided, total) from a device build's build_info"""
    m = re.match(r"device(?: \(forward\))?: (\d+) of (\d+) ", info)
    return (int(m.group(1)), int(m.group(2))) if m else (0, 0)


def run_case(bb, torch, pair, lens, globe, zoom, shape, k, max_fov, max_vfov, table):
    dev, ref = pair
    w, h, ps = shape
    rubix = k % 2 == 1
    grid = OTHER_GRID if k % 4 == 3 else DEFAULT_GRID
    for fe in pair:
        fe.set_rubixgrid(*grid)
        fe.command(f"f_globe {globe}")
        fe.command(f"f_lens {lens}")
        fe.command(zoom)
        fe.set_rubix(rubix)
    what = (lens, globe, zoom, shape, rubix, grid)
    got = build(bb, dev, w, h, ps, threads=0)
    info = dev.build_info
    want = build(bb, ref, w, h, ps, threads=-1)
    assert got[0] == want[0], what + (got[0], want[0], info)
    if refused_past_the_limit(zoom, max_fov, max_vfov):
        assert got[0] == bb.E_ZOOM, what
    assert got[4] == want[4], what + (got[4], want[4])
    assert got[5] == want[5], what + (np.frombuffer(got[5]), np.frombuffer(want[5]))
    assert np.array_equal(got[1], want[1]), what + (int((got[1] != want[1]).sum()), info)
    assert np.array_equal(got[2], want[2]), what + (info,)
    assert got[3] == want[3], what
    if got[0]:
        # a refused zoom publishes the empty map, as the reference renders it, on both paths; an export refuses it too
        assert (got[1] == -1).all(), what
        if dev.map_type == 1 and got[0] == bb.E_ZOOM:
            d = torch.zeros((h, w, 3), dtype=torch.float32, device="cuda")
            for call in (lambda: ref.raymap(w, h), lambda: dev.raymap(w, h, out=d)):
                with pytest.raises(bb.BlinkyError) as e:
                    call()
                assert e.value.code == bb.E_ZOOM, what
        return
    # the path: the documented fallback is an untranslatable lens (debug's nil tests)
    if lens in TRANSLATABLE:
        assert info.startswith("device:"), what + (info,)
    elif lens in FORWARD_ONLY:
        assert info.startswith("device (forward):"), what + (info,)
    else:
        assert lens == "debug" and info.startswith("host (") and "nil" in info, what + (info,)
    und, total = undecided_share(info)
    table.append((lens, globe, zoom, shape, und, total, float(np.frombuffer(got[5])[0])))
    # the export, for an inverse lens
    if dev.map_type == 1 and lens in TRANSLATABLE:
        with np.errstate(all="ignore"):
            host_rays = ref.raymap(w, h)
        d = torch.full((h, w, 3), 12345.0, dtype=torch.float32, device="cuda")
        dev.raymap(w, h, out=d)
        assert dev.build_info.startswith("ray export, device: "), what + (dev.build_info,)
        assert_same_rays(d.cpu().numpy(), host_rays, what)


def report(table, lens, seconds, ncases):
    rows = [r for r in table if r[5] and r[4] > 0.01 * r[5]]
    print(f"\n{lens}: {ncases} cases, {seconds:.1f} s")
    for lens_, globe, zoom, shape, und, total, scale in rows:
        print(f"  {globe:12s} {zoom:12s} {'x'.join(map(str, shape)):12s} {und:7d} of {total:7d} ({100.0 * und / total:5.1f} %)  "
              f"scale {scale:.6g}")


@pytest.mark.parametrize("lens", ALL_LENSES)
def test_device_build_and_export_over_the_zoom_sweep(bb, torch, pair, lens):
    t0 = time.time()
    dev, ref = pair
    for fe in pair:
        fe.command("f_globe cube")
    max_fov, max_vfov = zoom_limits(ref, lens)
    table = []
    k = 0
    # lens-major: the lens's units stay in the NVRTC cache for all of its zooms and globes
    for zoom in zooms(max_fov, max_vfov):
        for shape in SHAPES:
            run_case(bb, torch, pair, lens, "cube", zoom, shape, k, max_fov, max_vfov, table)
            k += 1
    for globe in REDUCED_GLOBES:
        for zoom, shape in reduced_cases(max_fov, max_vfov):
            run_case(bb, torch, pair, lens, globe, zoom, shape, k, max_fov, max_vfov, table)
            k += 1
    report(table, lens, time.time() - t0, k)
    assert len(table) >= 20, (lens, len(table))
    # flagged pixels near a pole cost time, not correctness (rectilinear at f_fov 180 flags every pixel but the centre):
    # only a sweep whose typical case is settled by the interpreter fails
    if lens in TRANSLATABLE + FORWARD_ONLY:
        shares = sorted(r[4] / r[5] for r in table if r[5])
        assert shares and shares[len(shares) // 2] <= 0.1, (lens, shares[len(shares) // 2])
