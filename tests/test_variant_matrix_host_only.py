"""The model and the reach of the warp-kernel matrix (test_gpu_variant_matrix.py), without a GPU.

1. expected_screen, the matrix's expected output, reproduces the compiled reference's frames, and agrees with a
   pixel-by-pixel statement of the same rule in RGBA, with per-frame tables and with keep_unmapped;
2. the matrix's kernels and variants are exactly the warp kernel instances the built library holds, so a new flag or
   kernel fails here until the matrix checks it."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_gpu_variant_matrix import KERNELS, VARIANTS, expected_screen

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_expected_screen_reproduces_the_reference_frames(bb, host, restate, palette):
    """frames_small.npz: the compiled reference rendered into a 160x120 screen filled with random bytes, view at (8, 6),
    unmapped pixels left alone — expected_screen of the oracle's frame, 8-bit with keep, is the same screen"""
    frames = np.load(os.path.join(G, "frames_small.npz"))
    W, H, PS = 128, 96, 48
    pm = restate.palmaps(palette)
    for key in frames.files:
        globe, lens, r = key.split("__")
        host.command(f"f_globe {globe}")
        host.command(f"f_lens {lens}")
        host.set_rubix(r == "rubix1")
        host.build_lensmap(W, H, PS, 8)
        idx, tint = host.lensmap()
        want8 = restate.render(idx, tint, bb.synthetic_faces(host.numplates, PS, 0), pm, r == "rubix1")[None]
        fill = np.random.default_rng(3).integers(0, 256, (120, 160), dtype=np.uint8)   # what Draw_TileClear left
        got = expected_screen(fill, want8, idx, nframes=1, x0=8, y0=6, rowbytes=160, frame_stride=120 * 160, keep=True)
        assert np.array_equal(got.reshape(120, 160), frames[key]), key


@pytest.mark.parametrize("rgba", ["8bit", "table", "tables"])
@pytest.mark.parametrize("keep", [False, True])
def test_expected_screen_pixel_by_pixel(rgba, keep):
    rng = np.random.default_rng(9)
    N, H, W, x0, y0, rowbytes, pad = 3, 5, 7, 3, 2, 48, 20
    bpp = 1 if rgba == "8bit" else 4
    frame_stride = (y0 + H + 1) * rowbytes + pad
    idx = np.where(rng.random((H, W)) < 0.6, rng.integers(0, 1000, (H, W)), -1).astype(np.int32)
    want8 = rng.integers(0, 256, (N, H, W), dtype=np.uint8)
    tables = rng.integers(0, 2**32, (N, 256), dtype=np.uint64).astype(np.uint32)
    fill = rng.integers(0, 256, N * frame_stride, dtype=np.uint8)
    got = expected_screen(fill, want8, idx, nframes=N, x0=x0, y0=y0, rowbytes=rowbytes, frame_stride=frame_stride, keep=keep,
                          table=tables[1] if rgba == "table" else None, tables=tables if rgba == "tables" else None)
    want = bytearray(fill.tobytes())
    for f in range(N):
        for y in range(H):
            for x in range(W):
                if keep and idx[y, x] < 0:
                    continue
                v = int(want8[f, y, x])
                if rgba != "8bit":
                    v = int(tables[f if rgba == "tables" else 1][v])
                at = f * frame_stride + (y0 + y) * rowbytes + (x0 + x) * bpp
                want[at:at + bpp] = v.to_bytes(bpp, "little")
    assert got.tobytes() == bytes(want)


INSTANCE = re.compile(r"(warp_ring_kernel|warp_tile_gather_kernel|warp_gather_kernel|warp_scalar_kernel)"
                      r"ILb([01])ELb([01])ELb([01])ELb([01])ELb([01])EE")


def test_the_matrix_covers_every_kernel_instance(bb):
    """The warp kernels' instances in libblinky_b200.so, from the names of their .text sections (template arguments
    <RUBIX, RGBA, KEEP, TABLES, LAYOUT>), are exactly KERNELS x VARIANTS of the matrix"""
    tool = shutil.which("cuobjdump") or next((p for p in ["/usr/local/cuda/bin/cuobjdump"] if os.path.exists(p)), None)
    if tool is None:
        pytest.skip("cuobjdump not found: cannot list the kernel instances of the built library")
    elf = subprocess.run([tool, "-elf", bb.LIB_PATH], check=True, capture_output=True, text=True).stdout
    found = set()
    for section in re.findall(r"\.text\.(\S+)", elf):
        m = INSTANCE.search(section)
        if m:
            found.add((m.group(1), tuple(int(b) for b in m.groups()[1:])))
    matrix = {(k, tuple(v)) for k in KERNELS for v in VARIANTS}
    assert len(matrix) == 96
    assert found == matrix, {"not in the matrix": sorted(found - matrix), "not in the library": sorted(matrix - found)}
