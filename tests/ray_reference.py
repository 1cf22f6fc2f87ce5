"""One frame of the ray warps by their rule, with no project kernel: blinky_warp_device_rays[_rgba] (k = 1, DESIGN §3d)
and blinky_warp_device_rays_supersampled (k = 2, 3, 4, DESIGN §3e).

1. Turn: the field turned in numpy float32 by the frame's matrix (test_gpu_ray_warp.turned).
2. Map: the turned rays mapped by the host blinky_set_raymap on a host-only context (Fisheye(device=None)) on the same
   globe, rubix state and grid; lensmap() gives each ray's texel idx (-1: unmapped) and tint (255: none).  A ray's
   texel does not depend on the view size, so a strip of a field, or the few distinct rays a tiled field repeats, may
   be mapped on their own.
3. Gather and colour: the face byte at plate_base[plate] + py * rowbytes + px (dense faces: plate * ps^2 + py * ps +
   px), the rubix LUT of palmaps() when rubix is on (tint 255: the identity), bg[y][x] of the output pixel for an
   unmapped sample, then the RGBA table (the shared one or the frame's own).
4. Average: for k > 1 each byte summed over the pixel's k x k samples in int64, written as (s + k^2 // 2) // k^2;
   with keep_unmapped a pixel is written exactly when one of its samples is mapped.  For k = 1 there is nothing to
   average, and 8-bit output is the palette index.

Also the arithmetic of the GPU limit cases (tests/test_gpu_ray_limits.py), which tests/test_ray_reference_host_only.py
asserts without a GPU."""
import numpy as np

from test_gpu_ray_warp import turned


class HostGlobe:
    """a host-only context on a globe, with the rubix state and grid of the device context it stands for"""

    def __init__(self, bb, palette, globe, rubix=False, grid=None):
        self.fe = bb.Fisheye(device=None, palette=palette)
        if grid:
            self.fe.set_rubixgrid(*grid)
        self.fe.command(f"f_globe {globe}")
        self.fe.set_rubix(rubix)
        self.rubix = rubix
        # rows 0-5: the plates' tint LUTs; row 6: the identity (tint 255)
        self.lut = np.vstack([self.fe.palmaps()[:6], np.arange(256, dtype=np.uint8)[None]])

    def close(self):
        self.fe.close()

    def texels(self, rays, ps, M=None):
        """(idx int64, tint uint8) of each ray of rays [..., 3] turned by M (None: as it is), by the host set_raymap"""
        shape = rays.shape[:-1]
        t = np.ascontiguousarray(rays if M is None else turned(rays, M), np.float32).reshape(1, -1, 3)
        with np.errstate(all="ignore"):
            self.fe.set_raymap(t, ps)
        idx, tint = self.fe.lensmap()
        return idx.astype(np.int64).reshape(shape), tint.reshape(shape)


def plate_bases(ps, layout=None):
    """(plate_base int64[6], rowbytes) of dense faces (layout None) or of a face layout (rowbytes, [(x, y), ...])"""
    if layout is None:
        return np.arange(6, dtype=np.int64) * ps * ps, ps
    rowbytes, origins = layout
    base = np.zeros(6, np.int64)
    for i, (x, y) in enumerate(origins):
        base[i] = int(y) * rowbytes + int(x)
    return base, rowbytes


def gather(faces, addr):
    """faces[addr]: faces a numpy array, or a CUDA uint8 tensor too large to copy to the host (gathered with torch)"""
    if isinstance(faces, np.ndarray):
        return faces[addr]
    import torch

    return faces[torch.from_numpy(np.ascontiguousarray(addr)).to(faces.device)].cpu().numpy()


def colour(g, idx, tint, faces, bg, k, ps, layout=None, table=None):
    """steps 3 and 4 for the texels (idx, tint) of the samples [k h, k w] of one frame: (pixels, written).  faces: the
    frame's bytes, uint8 1-D; bg: uint8 [h, w]; table: uint32[256] (RGBA) or None (8-bit, k = 1 only).  pixels:
    uint8 [h, w] (8-bit) or [h, w, 4] (RGBA bytes); written: bool [h, w], the pixels keep_unmapped writes."""
    kh, kw = idx.shape
    h, w = kh // k, kw // k
    assert (h * k, w * k) == (kh, kw) and bg.shape == (h, w)
    mapped = idx >= 0
    i = np.where(mapped, idx, 0)
    plate, rest = np.divmod(i, ps * ps)
    py, px = np.divmod(rest, ps)
    base, rowbytes = plate_bases(ps, layout)
    b = gather(faces, np.where(mapped, base[plate] + py * rowbytes + px, 0))
    if g.rubix:
        b = g.lut[np.where(tint == 255, 6, tint), b]
    b = np.where(mapped, b, np.repeat(np.repeat(bg, k, 0), k, 1)).astype(np.uint8)
    written = mapped.reshape(h, k, w, k).any(axis=(1, 3))
    if table is None:
        assert k == 1, "8-bit output is not averaged"
        return b, written
    c = np.asarray(table, np.uint32)[b].view(np.uint8).reshape(h, k, w, k, 4)
    s = c.astype(np.int64).sum(axis=(1, 3))
    return ((s + k * k // 2) // (k * k)).astype(np.uint8), written


def frame(g, field, M, faces, bg, k, ps, layout=None, table=None):
    """one frame of the warp of field [k h, k w, 3] turned by M: (pixels, written) as colour() gives them"""
    idx, tint = g.texels(field, ps, M)
    return colour(g, idx, tint, faces, bg, k, ps, layout, table)


# ---- tiled fields ------------------------------------------------------------------------------------------------

# The fields past 4 GiB repeat a small set of distinct rays with a period that divides neither a row of any of them nor
# 2^32 / 12 (a wrapped byte offset of a ray lands on another ray), so that the reference maps only the small set.
PERIOD = 1021   # prime


def tiled_texels(base_idx, base_tint, first, rows, fw, offset=0):
    """(idx, tint) [rows, fw] of the field rows first.. of a field fw rays wide that repeats the PERIOD rays whose
    texels are base_idx / base_tint from ray `offset` on: field pixel p holds ray (p + offset) % PERIOD"""
    p = (np.arange(first, first + rows, dtype=np.int64)[:, None] * fw + np.arange(fw, dtype=np.int64)[None] + offset) % PERIOD
    return base_idx[p], base_tint[p]


def fill_tiled(torch, dst, base, offset=0):
    """dst (a contiguous CUDA float32 [..., 3] tensor) := the tiling of base [PERIOD, 3] from ray `offset` on"""
    flat = dst.view(-1, 3)
    n = flat.shape[0]
    d = torch.as_tensor(np.roll(base, -offset, axis=0)).cuda()
    full = n // PERIOD
    if full:
        flat[: full * PERIOD].view(full, PERIOD, 3).copy_(d.expand(full, PERIOD, 3))
    flat[full * PERIOD:].copy_(d[: n - full * PERIOD])


# ---- the arithmetic of the GPU limit cases -----------------------------------------------------------------------

GiB4 = 1 << 32
MAX_PITCH = 1 << 26

# view shapes (w, h), run at k = 1, 2, 3, 4
SHAPES = [(1, 1), (3, 2), (1, 257), (257, 1), (255, 3), (97, 61), (1000, 8), (8, 640), (65600, 2), (2, 65600)]
THREADS = 256   # ray_warp.cu kRayThreads
MARGIN_ROWS = 256

# one limit at a time, for k = 1 (RGBA) and k = 4 (test_gpu_ray_limits.test_past_4_gib)
LIMIT_VIEW = (40, 24)                         # (w, h) of the small views
OUT_STRIDE = (1 << 30) + (1 << 16)            # frame 4 of 5 starts past 2^32
OUT_FRAMES = 5
PITCH_ROWS = 72                               # rows of a view at pitch 2^26: rows 64.. start past 2^32
FACE_STRIDE = GiB4 + 4099                     # frame 1's faces start past 2^32
PLATE_ROWBYTES = 1 << 16                      # a face layout whose plate 5 sits at row PLATE_Y, x PLATE_X
PLATE_Y, PLATE_X = (1 << 16) + 1, 7
RAY_STRIDE = GiB4 + 4 * 1001                  # bytes between frames' fields, tables and matrices: past 2^32 at f = 1
XFORM_STRIDE = GiB4 + 4 * 7
TABLE_STRIDE = GiB4 + 4 * 256 * 3
BIG_VIEW = (6144, 3648)                       # k = 4: a single field of more than 4 GiB

# the 31-bit field pixel index of the supersampled kernel, k = 4
FIELD_LIMIT_K = 4
REFUSED_VIEW = (16384, 8192)                  # k^2 W H = 2^31
TAKEN_VIEW = (16384, 8191)                    # k^2 W H = 2^31 - 2^18
# the far strides: frame 2 of 3 starts past 2^34 bytes, where the products f * ray_floats, f * xform_floats and
# f * table_words pass 2^32 (a table stride is at most 16 GB: the words between tables fit 32 bits)
FAR_STRIDE = (1 << 33) + 16
FAR_FRAMES = 3

# batches
MAX_FRAMES = 65535
ODD_BATCH = 997


def field_bytes(k, w, h):
    return 12 * k * k * w * h
