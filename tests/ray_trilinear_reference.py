"""One frame of the trilinear ray warp (blinky_warp_device_rays_trilinear, DESIGN §3g) by its rule, with no project kernel,
built on tests/ray_bilinear_reference.py:

1. Pyramid, in numpy integers: level 0's colour of each texel of every plate of the globe (the face byte, through the
   plate's rubix LUT when rubix is on and the texel is off the grid, then the frame's table), and each level L >= 1 the
   per-byte (sum of the clamped 2 x 2 block of level L - 1 + 2) >> 2, in the scratch layout (level-major, then plate,
   then rows of uint32 RGBA words).
2. Per pixel, the header (csrc/ray_texel.h behind the shim below, compiled with g++ -ffp-contract=off; the host-only
   tests pin its functions to an independent numpy restatement): mapping and plate, the footprint rho^2
   (ray_footprint2 over the turned, normalised neighbour rays), L and w (ray_level), and the bilinear positions on
   levels L and L + 1 (ray_bilinear_level).  Mapped-ness and plate are checked against the host set_raymap.
3. Taps, blends and the mix of the two levels in numpy: level 0's taps as ray_bilinear_reference takes them, level L's
   from the pyramid; per byte ((C00 (256 - wx) + C10 wx) (256 - wy) + (C01 (256 - wx) + C11 wx) wy + 32768) >> 16,
   then (C_L (256 - w) + C_L+1 w + 128) >> 8; an unmapped pixel takes the table colour of its background."""
import ctypes
import os
import subprocess

import numpy as np

import ray_bilinear_reference as br
import ray_reference as rr
from test_device_emulation import GRID
from test_ray_warp_host_only import params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = r"""
#include "ray_texel.h"
using namespace blinky;
// per pixel of a w x h field turned by M (nullptr: as it is): out[13] = mapped, plate, L, w, then (x0, y0, wx, wy) on
// level L and on level L + 1 (zeros at L = lmax); rho2 the footprint.  Unmapped: mapped = 0, the rest 0.
extern "C" void trilinear(const LensBuildParams *P, const float *M, const float *rays, int w, int h, int lmax, int32_t *out, double *rho2) {
    int size[kRayMaxLevels];
    uint64_t off[kRayMaxLevels], bytes;
    ray_pyramid_levels(P->platesize, P->numplates, size, off, &bytes);
    const auto turned = [&](long at, float t[3]) {
        const float *r = rays + 3 * at;
        t[0] = r[0], t[1] = r[1], t[2] = r[2];
        if (M) turn_ray(M, r, t);
    };
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            const long i = static_cast<long>(y) * w + x;
            int32_t *o = out + 13 * i;
            for (int k = 0; k < 13; ++k) o[k] = 0;
            rho2[i] = 0;
            float n[3];
            turned(i, n);
            int plate, px, py;
            double u, v;
            if (!ray_texel_uv(*P, n, &plate, &px, &py, &u, &v)) continue;
            float nb[4][3];
            const float *ptr[4] = {nullptr, nullptr, nullptr, nullptr};
            const bool have[4] = {x + 1 < w, x > 0, y + 1 < h, y > 0};
            const long at[4] = {i + 1, i - 1, i + w, i - w};
            for (int k = 0; k < 4; ++k)
                if (have[k]) {
                    turned(at[k], nb[k]);
                    ray_normalize3(nb[k]);
                    ptr[k] = nb[k];
                }
            const double r2 = ray_footprint2(*P, plate, n, ptr[0], ptr[1], ptr[2], ptr[3]);
            int L, wt;
            ray_level(r2, lmax, &L, &wt);
            o[0] = 1, o[1] = plate, o[2] = L, o[3] = wt;
            rho2[i] = r2;
            ray_bilinear_level(u, v, size[L], &o[4], &o[5], &o[6], &o[7]);
            if (L < lmax) ray_bilinear_level(u, v, size[L + 1], &o[8], &o[9], &o[10], &o[11]);
        }
}
// ray_plate_project of n normalised rays onto one plate: ok[i], a[i], b[i]
extern "C" void project(const LensBuildParams *P, int plate, const float *rays, size_t n, uint8_t *ok, double *a, double *b) {
    for (size_t i = 0; i < n; ++i) {
        a[i] = b[i] = -7;
        ok[i] = ray_plate_project(*P, plate, rays + 3 * i, &a[i], &b[i]);
    }
}
// ray_footprint2 of a sample n with neighbours (has[k] = 0: that neighbour is missing), k = xf, xb, yf, yb
extern "C" void footprint(const LensBuildParams *P, const int *plate, const float *n, const float *nb, const uint8_t *has, size_t count, double *rho2) {
    for (size_t i = 0; i < count; ++i) {
        const float *q[4];
        for (int k = 0; k < 4; ++k) q[k] = has[4 * i + k] ? nb + 12 * i + 3 * k : nullptr;
        rho2[i] = ray_footprint2(*P, plate[i], n + 3 * i, q[0], q[1], q[2], q[3]);
    }
}
// ray_on_rubix_line of columns 0..n-1
extern "C" void line(const LensBuildParams *P, int n, uint8_t *out) {
    for (int t = 0; t < n; ++t) out[t] = ray_on_rubix_line(*P, t);
}
extern "C" void level(const double *rho2, size_t n, int lmax, int32_t *L, int32_t *w) {
    for (size_t i = 0; i < n; ++i) ray_level(rho2[i], lmax, &L[i], &w[i]);
}
extern "C" int pyramid(int ps, int nplates, int32_t *size, uint64_t *off, uint64_t *bytes) {
    int s[kRayMaxLevels];
    const int lmax = ray_pyramid_levels(ps, nplates, s, off, bytes);
    for (int l = 0; l <= lmax; ++l) size[l] = s[l];
    return lmax;
}
"""


def compile_shim(directory):
    """the shim above as a ctypes library built in `directory`"""
    src = os.path.join(str(directory), "trilinear_shim.cpp")
    so = os.path.join(str(directory), "trilinear_shim.so")
    with open(src, "w") as f:
        f.write(SHIM)
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-Wall", "-Wextra", "-shared", "-fPIC", "-I",
                        os.path.join(ROOT, "blinky_b200", "csrc"), "-o", so, src], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:3000]
    lib = ctypes.CDLL(so)
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    lib.trilinear.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp]
    lib.project.argtypes = [vp, ctypes.c_int, vp, sz, vp, vp, vp]
    lib.footprint.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.level.argtypes = [vp, sz, ctypes.c_int, vp, vp]
    lib.line.argtypes = [vp, ctypes.c_int, vp]
    lib.pyramid.argtypes = [ctypes.c_int, ctypes.c_int, vp, vp, vp]
    return lib


# ---- the pyramid's layout, restated -------------------------------------------------------------------------------

def level_sizes(ps):
    """[s_0 = ps, s_1, ..., s_lmax = 1]"""
    sizes = [ps]
    while sizes[-1] > 1:
        sizes.append((sizes[-1] + 1) >> 1)
    return sizes


def pyramid_layout(ps, nplates):
    """(sizes, offsets of levels 1..lmax in bytes (offsets[0] = 0), B rounded up to 256, the unrounded total)"""
    sizes = level_sizes(ps)
    offs, at = [0], 0
    for s in sizes[1:]:
        offs.append(at)
        at += 4 * nplates * s * s
    return sizes, offs, (at + 255) // 256 * 256, at


def header_pyramid(lib, ps, nplates):
    """ray_pyramid_levels through the shim: (lmax, sizes, offsets, bytes)"""
    size = np.zeros(14, np.int32)
    off = np.zeros(14, np.uint64)
    b = ctypes.c_uint64(0)
    lmax = lib.pyramid(ps, nplates, size.ctypes.data, off.ctypes.data, ctypes.byref(b))
    return lmax, size[: lmax + 1].tolist(), off[: lmax + 1].tolist(), b.value


def header_trilinear(lib, p, M, field, lmax):
    """(int32 [h * w, 13], rho2 float64 [h * w]) of the shim's trilinear() over field [h, w, 3] turned by M"""
    h, w = field.shape[:2]
    flat = np.ascontiguousarray(field, np.float32)
    out = np.zeros((h * w, 13), np.int32)
    rho2 = np.zeros(h * w, np.float64)
    m = None if M is None else np.ascontiguousarray(M, np.float32)
    lib.trilinear(ctypes.byref(p), None if m is None else m.ctypes.data, flat.ctypes.data, w, h, lmax, out.ctypes.data, rho2.ctypes.data)
    return out, rho2


# ---- colours ------------------------------------------------------------------------------------------------------

def down(c):
    """the next level of colours c uint8 [..., s, s, 4]: per byte (sum of the clamped 2 x 2 block + 2) >> 2"""
    s = c.shape[-2]
    if s % 2:
        c = np.concatenate([c, c[..., -1:, :, :]], axis=-3)
        c = np.concatenate([c, c[..., :, -1:, :]], axis=-2)
    t = c.astype(np.uint16)
    total = t[..., 0::2, 0::2, :] + t[..., 0::2, 1::2, :] + t[..., 1::2, 0::2, :] + t[..., 1::2, 1::2, :]
    return ((total + 2) >> 2).astype(np.uint8)


def blend(C, wx, wy):
    """C[a, b] int64 [n, 4] of the taps (x0 + a, y0 + b), wx, wy int64 [n]: the bilinear blend per byte"""
    ux, uy, wx, wy = (256 - wx)[:, None], (256 - wy)[:, None], wx[:, None], wy[:, None]
    return ((C[0, 0] * ux + C[1, 0] * wx) * uy + (C[0, 1] * ux + C[1, 1] * wx) * wy + 32768) >> 16


class TrilinearGlobe(br.BilinearGlobe):
    """a BilinearGlobe (set_raymap on a host-only context, rubix LUTs) with the trilinear shim"""

    def __init__(self, bb, palette, globe, lib, rubix=False, grid=None):
        super().__init__(bb, palette, globe, None, rubix, grid)
        self.lib = lib
        self.nplates = self.fe.numplates

    def grid_line(self, ps):
        """ray_on_rubix_line of every column (row) of a plate of ps texels, bool [ps]"""
        p = params(self.fe, 1, 1, ps, self.grid)
        line = np.zeros(ps, np.uint8)
        self.lib.line(ctypes.byref(p), ps, line.ctypes.data)
        return line.astype(bool)

    def level0(self, faces, ps, plate, table, layout=None):
        """colours uint8 [ps, ps, 4] of level 0 of one plate, gathered a band of rows at a time"""
        base, rowbytes = rr.plate_bases(ps, layout)
        tab = np.asarray(table, np.uint32)
        out = np.empty((ps, ps, 4), np.uint8)
        xs = np.arange(ps, dtype=np.int64)
        line = self.grid_line(ps) if self.rubix else None
        for r0 in range(0, ps, 512):
            ys = np.arange(r0, min(ps, r0 + 512), dtype=np.int64)
            byte = rr.gather(faces, base[plate] + ys[:, None] * rowbytes + xs[None, :])
            if self.rubix:
                byte = np.where(~(line[None, :] | line[ys][:, None]), self.lut[plate][byte], byte)
            out[r0:r0 + len(ys)] = tab[byte].view(np.uint8).reshape(len(ys), ps, 4)
        return out

    def pyramid(self, faces, ps, table, layout=None):
        """[None, level 1 uint8 [nplates, s_1, s_1, 4], ..., level lmax]"""
        levels = [None] + [[] for _ in level_sizes(ps)[1:]]
        for plate in range(self.nplates):
            c = self.level0(faces, ps, plate, table, layout)
            for L in range(1, len(levels)):
                c = down(c)
                levels[L].append(c)
        return [None] + [np.stack(lv) for lv in levels[1:]]

    @staticmethod
    def scratch_bytes(levels):
        """the pyramid as the warp writes it to a frame's scratch: levels 1..lmax back to back (without the rounding)"""
        return np.concatenate([lv.reshape(-1) for lv in levels[1:]]) if len(levels) > 1 else np.zeros(0, np.uint8)

    def frame(self, field, M, faces, bg, ps, layout=None, table=None):
        """one frame of the trilinear warp of field [h, w, 3] turned by M: (pixels uint8 [h, w, 4], written bool [h, w],
        levels (pyramid()), per-pixel int32 [h * w, 13] and rho2 of the shim)"""
        h, w = field.shape[:2]
        assert bg.shape == (h, w)
        tab = np.asarray(table, np.uint32)
        idx, _ = self.texels(field, ps, M)
        mapped = (idx >= 0).reshape(-1)
        sizes = level_sizes(ps)
        lmax = len(sizes) - 1
        p = params(self.fe, w, h, ps, self.grid)
        s, rho2 = header_trilinear(self.lib, p, M, field, lmax)
        assert np.array_equal(s[:, 0] == 1, mapped), "the trilinear sample maps exactly what set_raymap maps"
        assert np.array_equal(s[mapped, 1], idx.reshape(-1)[mapped] // (ps * ps)), "on the same plate"
        levels = self.pyramid(faces, ps, tab, layout)
        plate = np.where(mapped, s[:, 1], 0).astype(np.int64)
        L, wt = s[:, 2].astype(np.int64), s[:, 3].astype(np.int64)
        base, rowbytes = rr.plate_bases(ps, layout)
        line = self.grid_line(ps) if self.rubix else None

        def colour_at(level_of, col):
            """the bilinear colour [n, 4] of each pixel on level level_of[i], positions from columns col..col+3"""
            out = np.zeros((len(plate), 4), np.int64)
            x0, y0, wx, wy = (s[:, col + c].astype(np.int64) for c in range(4))
            for lv in np.unique(level_of[mapped & (level_of >= 0)]):
                sel = mapped & (level_of == lv)
                sz = sizes[lv]
                xs = (np.maximum(x0[sel], 0), np.minimum(x0[sel] + 1, sz - 1))
                ys = (np.maximum(y0[sel], 0), np.minimum(y0[sel] + 1, sz - 1))
                C = {}
                for a in (0, 1):
                    for b in (0, 1):
                        if lv == 0:
                            byte = rr.gather(faces, base[plate[sel]] + ys[b] * rowbytes + xs[a]).astype(np.int64)
                            if self.rubix:
                                byte = np.where(~(line[xs[a]] | line[ys[b]]), self.lut[plate[sel], byte], byte)
                            C[a, b] = tab[byte].view(np.uint8).reshape(-1, 4).astype(np.int64)
                        else:
                            C[a, b] = levels[lv][plate[sel], ys[b], xs[a]].astype(np.int64)
                out[sel] = blend(C, wx[sel], wy[sel])
            return out

        c = colour_at(L, 4)
        mix = mapped & (wt > 0)
        if mix.any():
            c1 = colour_at(np.where(mix, L + 1, -1), 8)
            c = np.where(mix[:, None], (c * (256 - wt)[:, None] + c1 * wt[:, None] + 128) >> 8, c)
        unmapped = tab[bg.reshape(-1)].view(np.uint8).reshape(-1, 4).astype(np.int64)
        pix = np.where(mapped[:, None], c, unmapped).astype(np.uint8).reshape(h, w, 4)
        return pix, mapped.reshape(h, w), levels, s, rho2
