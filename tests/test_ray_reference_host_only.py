"""tests/ray_reference.py without a GPU: pinned to a literal per-sample loop over the host blinky_set_raymap, and the
arithmetic of the GPU limit cases (tests/test_gpu_ray_limits.py) asserted, so that no later edit shrinks a case below
the limit it is there for."""
import math

import numpy as np
import pytest

import ray_reference as rr
from test_gpu_ray_warp import matrices, turned

PS = 8
GRID = (2, 3.0, 1.0)


def loop_frame(g, field, M, faces, bg, k, ps, layout, table):
    """one frame, sample by sample: each ray turned and installed alone as a 1 x 1 ray map"""
    h, w = bg.shape
    lut = g.fe.palmaps()
    origins = None if layout is None else layout[1]
    rowbytes = ps if layout is None else layout[0]
    out = np.zeros((h, w, 4) if table is not None else (h, w), np.uint8)
    written = np.zeros((h, w), bool)
    halves = 0
    for y in range(h):
        for x in range(w):
            sums = [0, 0, 0, 0]
            for j in range(k):
                for i in range(k):
                    ray = field[k * y + j, k * x + i][None, None]
                    t = ray if M is None else turned(ray, M)
                    with np.errstate(all="ignore"):
                        g.fe.set_raymap(np.ascontiguousarray(t, np.float32), ps)
                    idx, tint = g.fe.lensmap()
                    idx, tint = int(idx[0, 0]), int(tint[0, 0])
                    if idx >= 0:
                        written[y, x] = True
                        plate, px, py = idx // (ps * ps), idx % ps, idx // ps % ps
                        ox, oy = (0, plate * ps) if origins is None else origins[plate]
                        b = int(faces[(oy + py) * rowbytes + ox + px])
                        if g.rubix and tint != 255:
                            b = int(lut[tint][b])
                    else:
                        b = int(bg[y, x])
                    if table is None:
                        out[y, x] = b
                    else:
                        c = int(table[b])
                        for ch in range(4):
                            sums[ch] += (c >> (8 * ch)) & 0xFF
            if table is not None:
                for ch in range(4):
                    out[y, x, ch] = math.floor(sums[ch] / (k * k) + 0.5)   # half up
                    halves += k % 2 == 0 and sums[ch] % (k * k) == k * k // 2
    return out, written, halves


def half_table(seed):
    """a table whose channels take two neighbouring values (0/1, 100/101, 254/255) and one random byte: averages of
    k x k samples often land exactly half-way"""
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 2, (256, 3))
    t = bits[:, 0] | (100 + bits[:, 1]) << 8 | (254 + bits[:, 2]) << 16 | rng.integers(0, 256, 256) << 24
    return t.astype(np.uint32)


@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("view", [(1, 1), (3, 2), (5, 7)])
@pytest.mark.parametrize("faces_form", ["dense", "layout"])
def test_reference_equals_the_per_sample_loop(bb, palette, k, view, faces_form):
    w, h = view
    layout = None if faces_form == "dense" else (2 * PS + 5, [(3 + (i % 2) * (PS + 1), 1 + (i // 2) * (PS + 2)) for i in range(6)])
    size = 6 * PS * PS if layout is None else (max(y for _, y in layout[1]) + PS) * layout[0]
    rng = np.random.default_rng(k * 100 + w)
    halves = 0
    for rubix in (False, True):
        g = rr.HostGlobe(bb, palette, "cube", rubix=rubix, grid=GRID if rubix else None)
        try:
            g.fe.command("f_lens panini")
            g.fe.command("f_fov 180")
            field = g.fe.raymap(k * w, k * h)
            flat = field.reshape(-1, 3)
            flat[::5] = rng.normal(size=flat[::5].shape).astype(np.float32)
            flat[2::7] = 0
            flat[3::11] = [np.inf, 0, 1]
            bg = rng.integers(0, 256, (h, w), dtype=np.uint8)
            xs = matrices(2, seed=w + k)
            # frame 0: the shared table; frame 1: its own table, built to land averages half-way
            tables = [np.asarray(rng.integers(0, 2**32, 256, dtype=np.uint32)), half_table(k)]
            for f in range(2):
                faces = rng.integers(0, 256, size, dtype=np.uint8)
                for table in ([tables[f]] if k > 1 else [None, tables[f]]):
                    pix, written = rr.frame(g, field, xs[f], faces, bg, k, PS, layout, table)
                    want, want_written, n_half = loop_frame(g, field, xs[f], faces, bg, k, PS, layout, table)
                    assert np.array_equal(pix, want), (rubix, f, table is None)
                    assert np.array_equal(written, want_written), (rubix, f)
                    halves += n_half
        finally:
            g.close()
    if k % 2 == 0 and w * h > 1:
        assert halves > 0, "no channel sum landed half-way: the rounding direction is not pinned"


def test_unmapped_pixels_and_keep():
    """written is exactly 'one of the k x k samples mapped'; unmapped samples take the pixel's background"""
    class G:
        rubix = False

    k, ps = 2, 4
    idx = np.full((4, 4), -1, np.int64)
    idx[0, 1] = 5              # pixel (0, 0): one mapped sample
    idx[2:, 2:] = 7            # pixel (1, 1): all four
    tint = np.full((4, 4), 255, np.uint8)
    faces = np.arange(6 * ps * ps, dtype=np.uint8)
    bg = np.array([[10, 20], [30, 40]], np.uint8)
    table = np.arange(256, dtype=np.uint32) * 0x01010101
    pix, written = rr.colour(G(), idx, tint, faces, bg, k, ps, table=table)
    assert written.tolist() == [[True, False], [False, True]]
    # (5 + 3 * 10 + 2) // 4 = 9; 20; 30; 7
    assert pix[..., 0].tolist() == [[9, 20], [30, 7]] and (pix == pix[..., :1]).all()


# ---- the arithmetic of the GPU limit cases -----------------------------------------------------------------------

def test_view_shapes_reach_their_limits():
    shapes = rr.SHAPES
    assert (1, 1) in shapes and any(w == 1 and h > 1 for w, h in shapes) and any(h == 1 and w > 1 for w, h in shapes)
    assert any(w % 2 == 1 and w > 1 for w, _ in shapes)
    assert max(w for w, _ in shapes) > 65536 and max(h for _, h in shapes) > 65536
    # a partial last CTA (pixels per thread) in every shape but 8 x 640
    partial = [s for s in shapes if s[0] * s[1] % rr.THREADS != 0]
    assert [s for s in shapes if s not in partial] == [(8, 640)]
    # a missing guard writes at most THREADS - 1 pixels past the view: inside the margin rows even for 1-pixel rows
    assert rr.MARGIN_ROWS >= rr.THREADS - 1


def test_offsets_past_4_gib():
    w, h = rr.LIMIT_VIEW
    assert (rr.OUT_FRAMES - 1) * rr.OUT_STRIDE > rr.GiB4 > (rr.OUT_FRAMES - 2) * rr.OUT_STRIDE
    assert rr.OUT_STRIDE % 16 == 0
    assert (rr.PITCH_ROWS - 1) * rr.MAX_PITCH >= rr.GiB4 and rr.MAX_PITCH == 1 << 26
    assert rr.FACE_STRIDE > rr.GiB4
    assert rr.PLATE_Y * rr.PLATE_ROWBYTES + rr.PLATE_X > rr.GiB4 and rr.PLATE_Y < 2**31 and rr.PLATE_ROWBYTES < 2**31
    for s in (rr.RAY_STRIDE, rr.XFORM_STRIDE, rr.TABLE_STRIDE):
        assert s > rr.GiB4 and s % 4 == 0
    for k in (1, 4):
        assert rr.RAY_STRIDE >= rr.field_bytes(k, w, h)
    assert rr.TABLE_STRIDE >= 1024 and rr.XFORM_STRIDE >= 36
    # about 9 GB at most for each case
    assert (rr.PITCH_ROWS - 1) * rr.MAX_PITCH < 9e9 and (rr.OUT_FRAMES - 1) * rr.OUT_STRIDE < 9e9
    bw, bh = rr.BIG_VIEW
    assert rr.field_bytes(4, bw, bh) > rr.GiB4 and 16 * bw * bh < 2**31
    # the last 64 rows of the big view hold the rays past 2^32 bytes
    assert (bh - 64) * 4 * 4 * bw * 12 < rr.GiB4


def test_the_tiling_period():
    p = rr.PERIOD
    assert all(p % q for q in range(2, int(p ** 0.5) + 1))
    widths = [k * w for k in (1, 2, 3, 4) for w, _ in rr.SHAPES] + [k * rr.LIMIT_VIEW[0] for k in (1, 4)] + [4 * rr.BIG_VIEW[0], 4 * rr.TAKEN_VIEW[0]]
    assert all(fw % p for fw in widths if fw >= p)
    assert (rr.GiB4 // 12) % p != 0 and rr.GiB4 % (12 * p) != 0


def test_the_31_bit_field_index():
    k = rr.FIELD_LIMIT_K
    W, H = rr.REFUSED_VIEW
    assert k * k * W * H == 2**31
    W, H = rr.TAKEN_VIEW
    n = k * k * W * H
    assert n == 2**31 - 2**18   # one row of 16384 pixels less: 16 * 16384 samples
    # the float index of the last samples passes 2^32: a 32-bit 3 * index wraps there
    assert 3 * (n - 1) >= 2**32
    # the far strides: the products f * floats (or words) pass 2^32 at the last frame, and the memory of the
    # 2^31 - 2^18 field holds them
    f = rr.FAR_FRAMES - 1
    assert f * (rr.FAR_STRIDE // 4) >= 2**32 and rr.FAR_STRIDE % 16 == 0 and rr.FAR_STRIDE // 4 <= 2**32 - 1
    assert f * rr.FAR_STRIDE + rr.field_bytes(4, *rr.LIMIT_VIEW) + 4096 <= 12 * n


def test_batches():
    assert rr.MAX_FRAMES == 65535
    assert rr.ODD_BATCH % 2 == 1 and all(rr.ODD_BATCH % q for q in range(2, 32))


def test_tiled_texels_and_fill():
    base_idx = np.arange(rr.PERIOD, dtype=np.int64) * 3
    base_tint = (np.arange(rr.PERIOD) % 7).astype(np.uint8)
    idx, tint = rr.tiled_texels(base_idx, base_tint, 2, 3, 500, offset=11)
    p = (np.arange(2 * 500, 5 * 500) + 11) % rr.PERIOD
    assert np.array_equal(idx.reshape(-1), base_idx[p]) and np.array_equal(tint.reshape(-1), base_tint[p])
