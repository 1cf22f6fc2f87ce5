"""One frame of the bilinear ray warp (blinky_warp_device_rays_bilinear, DESIGN §3f) by its rule, with no project kernel,
built on tests/ray_reference.py:

1. Turn and map: the field turned in numpy float32, each ray mapped by the host blinky_set_raymap on a host-only
   context (ray_reference.HostGlobe), which decides whether a sample is mapped and on which plate.
2. Position: ray_bilinear and ray_on_rubix_line of csrc/ray_texel.h, compiled with g++ -ffp-contract=off behind a small
   shim (tests/test_ray_bilinear_host_only.py pins both to an independent numpy restatement): (x0, y0, wx, wy) per sample
   and the grid test of every texel column and row.
3. Taps, LUTs, tables, blend and average in numpy: the taps (x0 | x0 + 1, y0 | y0 + 1) clamped to [0, ps - 1] on the
   sample's plate, each tap's byte through the plate's rubix LUT when rubix is on and the tap is off the grid, then the
   frame's table; per byte ((C00 (256 - wx) + C10 wx) (256 - wy) + (C01 (256 - wx) + C11 wx) wy + 32768) >> 16; an
   unmapped sample takes the table colour of the output pixel's background; k x k samples are averaged as
   ray_reference.colour averages them, (s + k^2 // 2) // k^2."""
import ctypes
import os
import subprocess

import numpy as np

import ray_reference as rr
from test_device_emulation import GRID
from test_ray_warp_host_only import params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = r"""
#include "ray_texel.h"
using namespace blinky;
// per ray: ray_entry's packed entry, and ray_bilinear's (mapped, plate, x0, y0, wx, wy) of the ray turned by M
extern "C" void samples(const LensBuildParams *P, const float *M, const float *rays, size_t n, uint32_t *entry, int32_t *out) {
    for (size_t i = 0; i < n; ++i) {
        const float *r = rays + 3 * i;
        entry[i] = ray_entry(*P, M, r);
        float t[3] = {r[0], r[1], r[2]};
        if (M) turn_ray(M, r, t);
        int32_t *o = out + 6 * i;
        o[1] = o[2] = o[3] = o[4] = o[5] = -7;
        o[0] = ray_bilinear(*P, t, &o[1], &o[2], &o[3], &o[4], &o[5]);
    }
}
// line[t] = ray_on_rubix_line(t) for t < n; with cell, cell[y * n + x] = ray_on_rubix_grid(x, y)
extern "C" void grid(const LensBuildParams *P, int n, uint8_t *line, uint8_t *cell) {
    for (int t = 0; t < n; ++t) line[t] = ray_on_rubix_line(*P, t);
    if (cell)
        for (int y = 0; y < n; ++y)
            for (int x = 0; x < n; ++x) cell[y * n + x] = ray_on_rubix_grid(*P, x, y);
}
"""


def compile_shim(directory):
    """the shim above as a ctypes library built in `directory`"""
    src = os.path.join(str(directory), "bilinear_shim.cpp")
    so = os.path.join(str(directory), "bilinear_shim.so")
    with open(src, "w") as f:
        f.write(SHIM)
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-Wall", "-Wextra", "-shared", "-fPIC", "-I",
                        os.path.join(ROOT, "blinky_b200", "csrc"), "-o", so, src], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:3000]
    lib = ctypes.CDLL(so)
    lib.samples.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]
    lib.grid.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def header_samples(lib, p, M, rays):
    """(ray_entry's entries uint32 [n], ray_bilinear's int32 [n, 6]) of rays [..., 3] turned by M (None: as they are)"""
    flat = np.ascontiguousarray(rays.reshape(-1, 3), np.float32)
    entry = np.zeros(len(flat), np.uint32)
    out = np.zeros((len(flat), 6), np.int32)
    m = None if M is None else np.ascontiguousarray(M, np.float32)
    lib.samples(ctypes.byref(p), None if m is None else m.ctypes.data, flat.ctypes.data, len(flat), entry.ctypes.data, out.ctypes.data)
    return entry, out


class BilinearGlobe(rr.HostGlobe):
    """a HostGlobe (set_raymap on a host-only context) with the shim for positions, on the grid it was made with"""

    def __init__(self, bb, palette, globe, lib, rubix=False, grid=None):
        super().__init__(bb, palette, globe, rubix, grid)
        self.lib = lib
        self.grid = grid or GRID

    def frame(self, field, M, faces, bg, k, ps, layout=None, table=None):
        """one frame of the bilinear warp of field [k h, k w, 3] turned by M: (pixels uint8 [h, w, 4], written bool
        [h, w]).  faces: the frame's bytes (numpy uint8 1-D, or a CUDA uint8 tensor); bg: uint8 [h, w]; table:
        uint32[256]."""
        kh, kw = field.shape[:2]
        h, w = kh // k, kw // k
        assert (h * k, w * k) == (kh, kw) and bg.shape == (h, w)
        idx, _ = self.texels(field, ps, M)
        mapped = (idx >= 0).reshape(-1)
        p = params(self.fe, kw, kh, ps, self.grid)
        _, s = header_samples(self.lib, p, M, field)
        assert np.array_equal(s[:, 0] == 1, mapped), "ray_bilinear maps exactly what set_raymap maps"
        assert np.array_equal(s[mapped, 1], idx.reshape(-1)[mapped] // (ps * ps)), "on the same plate"
        plate = np.where(mapped, s[:, 1], 0).astype(np.int64)
        x0, y0, wx, wy = (np.where(mapped, s[:, c], 0).astype(np.int64) for c in (2, 3, 4, 5))
        xs = (np.maximum(x0, 0), np.minimum(x0 + 1, ps - 1))
        ys = (np.maximum(y0, 0), np.minimum(y0 + 1, ps - 1))
        base, rowbytes = rr.plate_bases(ps, layout)
        if self.rubix:
            line = np.zeros(ps, np.uint8)
            self.lib.grid(ctypes.byref(p), ps, line.ctypes.data, None)
            line = line.astype(bool)
        tab = np.asarray(table, np.uint32)
        C = {}
        for a in (0, 1):
            for b in (0, 1):
                byte = rr.gather(faces, np.where(mapped, base[plate] + ys[b] * rowbytes + xs[a], 0)).astype(np.int64)
                if self.rubix:
                    off = ~(line[xs[a]] | line[ys[b]])
                    byte = np.where(off, self.lut[plate, byte], byte)
                C[a, b] = tab[byte].view(np.uint8).reshape(-1, 4).astype(np.int64)
        ux, uy = (256 - wx)[:, None], (256 - wy)[:, None]
        wx, wy = wx[:, None], wy[:, None]
        blend = ((C[0, 0] * ux + C[1, 0] * wx) * uy + (C[0, 1] * ux + C[1, 1] * wx) * wy + 32768) >> 16
        bgk = np.repeat(np.repeat(bg, k, 0), k, 1).reshape(-1)
        unmapped = tab[bgk].view(np.uint8).reshape(-1, 4).astype(np.int64)
        c = np.where(mapped[:, None], blend, unmapped).reshape(h, k, w, k, 4)
        total = c.sum(axis=(1, 3))
        written = mapped.reshape(h, k, w, k).any(axis=(1, 3))
        return ((total + k * k // 2) // (k * k)).astype(np.uint8), written
