"""Face layouts (blinky_set_face_layout) without a GPU: the argument checks, the host-only context's refusal of the
warps, f_saveglobe reading plates out of an atlas, the offset split the kernels use (face_layout.h, compiled here with
g++), and the tile plan interpreted with layout addressing against the reference's render_lensmap."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMPTY, BOX, GATHER, BOX_FULL = 0, 1, 2, 3
BOX_BLOCK = 2048 + 128


def atlas(faces, rowbytes, origins, rows, seed=0):
    """[N, rows, rowbytes] surfaces holding plate i of each frame at byte x, row y = origins[i]; random gap bytes"""
    faces = faces.reshape(-1, *faces.shape[-3:])
    n, p, ps, _ = faces.shape
    out = np.random.default_rng(seed).integers(0, 256, (n, rows, rowbytes), dtype=np.uint8)
    for i in range(p):
        x, y = origins[i]
        out[:, y:y + ps, x:x + ps] = faces[:, i]
    return out


def atlas_3x2(ps, pad=0, gap=0):
    """3x2 atlas of six plates, `gap` bytes / rows between them, rows padded by `pad` bytes"""
    origins = [(c * (ps + gap), r * (ps + gap)) for r in range(2) for c in range(3)]
    return 3 * ps + 2 * gap + pad, origins, 2 * ps + gap


def test_set_face_layout_argument_errors(bb, host):
    lib, ctx = host._lib, host._ctx
    org = (ctypes.c_int32 * 12)(*[0, 0] * 6)
    assert lib.blinky_set_face_layout(ctx, -1, org, 6) == bb.E_INVALID
    assert lib.blinky_set_face_layout(ctx, 64, None, 6) == bb.E_INVALID
    assert lib.blinky_set_face_layout(ctx, 64, org, 0) == bb.E_INVALID
    assert lib.blinky_set_face_layout(ctx, 64, org, 7) == bb.E_INVALID
    for k in range(12):
        bad = (ctypes.c_int32 * 12)(*[3] * 12)
        bad[k] = -1
        assert lib.blinky_set_face_layout(ctx, 64, bad, 6) == bb.E_INVALID
    assert lib.blinky_set_face_layout(ctx, 64, org, 6) == bb.OK
    assert lib.blinky_set_face_layout(ctx, 0, None, 0) == bb.OK   # dense again; origins are not read
    with pytest.raises(bb.BlinkyError) as e:
        host.set_face_layout(32, [(0, 0), (-16, 0)])
    assert e.value.code == bb.E_INVALID
    assert host.face_layout is None
    host.set_face_layout(48, [(0, 0), (16, 40)])
    assert host.face_layout == (48, [(0, 0), (16, 40)])
    host.set_face_layout()
    assert host.face_layout is None


def test_host_only_context_refuses_layout_warps(bb, host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.build_lensmap(64, 48, 32)
    rowbytes, origins, rows = atlas_3x2(32, pad=16)
    host.set_face_layout(rowbytes, origins)
    surf = atlas(bb.synthetic_faces(6, 32, 0), rowbytes, origins, rows)
    calls = [lambda: host.warp(0, 0, nframes=2, face_stride=rows * rowbytes),
             lambda: host.warp(0, 0, nframes=1, rgba=True),
             lambda: host.warp_view(0, 0, x0=4, y0=2, rowbytes=80, nframes=2, keep_unmapped=True),
             lambda: host.warp_host(surf)]
    for call in calls:
        with pytest.raises(bb.BlinkyError) as e:
            call()
        assert e.value.code == bb.E_NODEVICE
    assert host.launch_count == 0


@pytest.mark.parametrize("globe", ["cube", "trism", "fast"])
def test_save_globe_from_an_atlas_writes_the_dense_bytes(bb, host, tmp_path, globe):
    w, h = 48, 40
    ps = 40
    for margins in (0, 1):
        host.command(f"f_globe {globe}")
        host.command("f_lens equirect")
        faces = bb.synthetic_faces(host.numplates, ps, 6)
        n = host.numplates
        # plates in a row with odd gaps and a padded pitch
        origins = [(3 + i * (ps + 5), 7 + (i % 2) * 3) for i in range(n)]
        rowbytes = origins[-1][0] + ps + 9
        surf = atlas(faces, rowbytes, origins, 7 + 3 + ps + 2)[0]
        for name, layout, data in (("dense", None, faces), ("atlas", (rowbytes, origins), surf)):
            os.makedirs(tmp_path / name, exist_ok=True)
            if layout:
                host.set_face_layout(*layout)
            host.command(f"f_saveglobe g{margins}_ {margins}")
            host.build_lensmap(w, h, ps)
            host.save_globe(data, str(tmp_path / name))
            host.set_face_layout()
        for i in range(n):
            a = open(tmp_path / "dense" / f"g{margins}_{i}.pcx", "rb").read()
            b = open(tmp_path / "atlas" / f"g{margins}_{i}.pcx", "rb").read()
            assert a == b, (globe, margins, i)
    # a layout without an origin for every plate, or one whose plates overhang the pitch, is refused
    host.command("f_globe cube")
    host.build_lensmap(w, h, ps)
    host.set_face_layout(2 * ps, [(0, 0), (ps, 0)])
    with pytest.raises(bb.BlinkyError) as e:
        host.save_globe(np.zeros((2 * ps, 2 * ps), np.uint8), str(tmp_path))
    assert e.value.code == bb.E_INVALID
    host.set_face_layout(2 * ps, [(0, 0), (ps + 1, 0)] * 3)
    with pytest.raises(bb.BlinkyError) as e:
        host.save_globe(np.zeros((2 * ps, 2 * ps), np.uint8), str(tmp_path))
    assert e.value.code == bb.E_INVALID


# ---- the offset split (face_layout.h) --------------------------------------------------------------------------------

SHIM = r"""
#include "face_layout.h"
using namespace blinky;
extern "C" void split(const uint32_t *ps, const uint32_t *off, size_t n, uint32_t *plate, uint32_t *py, uint32_t *px) {
    for (size_t i = 0; i < n; ++i) {
        const FastDiv d2 = make_fastdiv(ps[i] * ps[i]), d1 = make_fastdiv(ps[i]);
        plate[i] = fastdiv(off[i], d2);
        const uint32_t rem = off[i] - plate[i] * ps[i] * ps[i];
        py[i] = fastdiv(rem, d1);
        px[i] = rem - py[i] * ps[i];
    }
}
extern "C" void texels(uint32_t ps, uint32_t rowbytes, const int32_t *origins, const uint32_t *off, size_t n, uint64_t *out) {
    FaceLayoutParams L = {};
    for (int i = 0; i < kLayoutPlates; ++i) L.plate_base[i] = uint64_t(origins[2 * i + 1]) * rowbytes + uint64_t(origins[2 * i]);
    L.rowbytes = rowbytes;
    L.ps = ps;
    L.ps2 = ps * ps;
    L.div_ps = make_fastdiv(ps);
    L.div_ps2 = make_fastdiv(ps * ps);
    for (size_t i = 0; i < n; ++i) out[i] = layout_texel(off[i], L);
}
"""


@pytest.fixture(scope="module")
def split_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("face_layout")
    src = d / "shim.cpp"
    src.write_text(SHIM)
    so = d / "shim.so"
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "blinky_b200", "csrc"), "-o", str(so), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(so))


def _split(lib, ps, off):
    ps, off = np.ascontiguousarray(ps, np.uint32), np.ascontiguousarray(off, np.uint32)
    out = [np.empty(off.size, np.uint32) for _ in range(3)]
    lib.split(ctypes.c_void_p(ps.ctypes.data), ctypes.c_void_p(off.ctypes.data), ctypes.c_size_t(off.size),
              *(ctypes.c_void_p(a.ctypes.data) for a in out))
    return out


def test_offset_split_is_exact_for_every_plate_size(split_lib):
    """every ps from 1 to 6688 (6 plates of 6688^2 texels fill the 28-bit index): offsets at plate and row
    boundaries, and random ones, against // and %"""
    rng = np.random.default_rng(11)
    all_ps, all_off = [], []
    for ps in range(1, 6689):
        ps2 = ps * ps
        top = min(6 * ps2, 1 << 28)
        k = np.arange(7, dtype=np.int64) * ps2
        rows = np.concatenate([np.arange(min(ps, 8)), rng.integers(0, ps, 8), [ps - 1]]).astype(np.int64) * ps
        plates = rng.integers(0, 6, rows.size) * ps2
        cand = np.concatenate([k - 1, k, k + 1, plates + rows - 1, plates + rows, plates + rows + 1, rng.integers(0, top, 24),
                               [top - 1]])
        cand = cand[(cand >= 0) & (cand < top)]
        all_ps.append(np.full(cand.size, ps, np.int64))
        all_off.append(cand)
    ps, off = np.concatenate(all_ps), np.concatenate(all_off)
    plate, py, px = _split(split_lib, ps, off)
    assert np.array_equal(plate, off // (ps * ps))
    assert np.array_equal(py, off % (ps * ps) // ps)
    assert np.array_equal(px, off % ps)
    assert off.size > 6688 * 60


def test_layout_texel_addresses_the_surface(split_lib):
    rng = np.random.default_rng(5)
    for ps, rowbytes, origins in ((16, 48, [(0, 0), (16, 0), (32, 0), (0, 16), (16, 16), (32, 16)]),
                                  (100, 331, [(3, 1), (103, 0), (220, 9), (0, 120), (117, 130), (231, 101)]),
                                  (6688, 3 * 6688 + 16, [(c * 6688, r * 6688) for r in range(2) for c in range(3)])):
        off = rng.integers(0, 6 * ps * ps, 20000).astype(np.uint32)
        org = np.ascontiguousarray(np.array(origins, np.int32).reshape(-1))
        out = np.empty(off.size, np.uint64)
        split_lib.texels(ctypes.c_uint32(ps), ctypes.c_uint32(rowbytes), ctypes.c_void_p(org.ctypes.data), ctypes.c_void_p(off.ctypes.data),
                         ctypes.c_size_t(off.size), ctypes.c_void_p(out.ctypes.data))
        o = off.astype(np.int64)
        plate, py, px = o // (ps * ps), o % (ps * ps) // ps, o % ps
        ox, oy = np.array(origins)[plate].T
        assert np.array_equal(out.astype(np.int64), (oy + py) * rowbytes + ox + px)


# ---- the tile plan read through a layout ------------------------------------------------------------------------------

def render_from_plan_with_layout(fe, surf, rowbytes, origins, palmaps, bg, rubix):
    """the tile plan interpreted the way the kernels do with a face layout: a BOX tile's TMA box is cut out of the
    surface at its plate-space origin plus the plate's origin (zero fill outside the surface, neighbouring texels
    where it overhangs its plate), a GATHER entry's offset is split into (plate, py, px)"""
    tiles, entries = fe.tile_plan()
    W, H, ps = fe.width, fe.height, fe.platesize
    rows = surf.shape[0]
    out = bg.copy()
    lut = np.concatenate([palmaps, np.arange(256, dtype=np.uint8)[None], np.arange(256, dtype=np.uint8)[None]])
    types = tiles["type"] & 3
    nbox = int(np.isin(types, (BOX, BOX_FULL)).sum())
    lanes = np.arange(32)
    org = np.array(origins, np.int64)
    for n, t in enumerate(tiles):
        x0, y0 = int(t["px"]), int(t["py"])
        ys, xs = min(32, H - y0), min(32, W - x0)
        ty = int(t["type"]) & 3
        if ty == EMPTY:
            continue
        if ty in (BOX, BOX_FULL):
            bw, bh = int(t["box_w16"]) * 16, int(t["box_h8"]) * 8
            plate, tile_tint = int(t["plate"]) & 7, (int(t["plate"]) >> 3) & 7
            bx, by = int(t["box_x"]) + origins[plate][0], int(t["box_y"]) + origins[plate][1]
            box = np.zeros((bh, bw), np.uint8)
            sy0, sy1 = max(by, 0), min(by + bh, rows)
            sx0, sx1 = max(bx, 0), min(bx + bw, rowbytes)
            if sy1 > sy0 and sx1 > sx0:
                box[sy0 - by:sy1 - by, sx0 - bx:sx1 - bx] = surf[sy0:sy1, sx0:sx1]
            blk = entries[n * BOX_BLOCK:(n + 1) * BOX_BLOCK]
            ent = blk[:2048].view("<u2").reshape(4, 32, 8)
            flags = blk[2048:].view("<u4")
            e = np.zeros((32, 32), np.uint16)
            tint = np.zeros((32, 32), np.int64)
            for i in range(32):
                r, c = (lanes >> 3) + 4 * (i >> 2), 4 * (lanes & 7) + (i & 3)
                e[r, c] = ent[i >> 3, lanes, i & 7]
                tint[r, c] = np.where((flags >> i) & 1, tile_tint, 6)
            valid = (e & 0x8000) != 0
            px = box.reshape(-1)[np.where(valid, (e & 0x3FFF).astype(np.int64), 0)]
        else:
            e = entries[int(t["entry_offset"]):int(t["entry_offset"]) + 4096].view("<u4").reshape(32, 32)
            valid = (e & 0x80000000) != 0
            off = np.where(valid, e & 0x0FFFFFFF, 0).astype(np.int64)
            plate, py, pxx = off // (ps * ps), off % (ps * ps) // ps, off % ps
            px = surf[org[plate, 1] + py, org[plate, 0] + pxx]
            tint = ((e >> 28) & 7).astype(np.int64)
        if rubix:
            px = lut[np.minimum(tint, 7), px]
        sub = out[y0:y0 + ys, x0:x0 + xs]
        sub[valid[:ys, :xs]] = px[:ys, :xs][valid[:ys, :xs]]
    assert nbox > 0 or ps % 16
    return out


@pytest.mark.parametrize("rubix", [False, True])
@pytest.mark.parametrize("globe,lens,zoom,size", [
    ("cube", "panini", "f_fov 180", (320, 240, 128)),
    ("cube", "fisheye1", "f_contain", (320, 200, 208)),
    ("cube", "quincuncial", "f_cover", (333, 201, 128)),
    ("trism", "hammer", "f_contain", (256, 160, 64)),
    ("fast", "stereographic", "f_fov 200", (256, 160, 96)),
])
def test_plan_read_through_a_layout_equals_reference_render(bb, host, restate, palette, globe, lens, zoom, size, rubix):
    w, h, ps = size
    host.command(f"f_globe {globe}")
    host.command(f"f_lens {lens}")
    host.command(zoom)
    host.set_rubix(rubix)
    host.build_lensmap(w, h, ps, threads=2)
    idx, tint = host.lensmap()
    faces = bb.synthetic_faces(host.numplates, ps, 5)
    bg = bb.synthetic_background(w, h)
    pm = restate.palmaps(palette)
    want = restate.render(idx, tint, faces, pm, rubix, background=bg)
    n = host.numplates
    for rowbytes, origins, rows in (atlas_3x2(ps, pad=16, gap=16), atlas_3x2(ps, pad=5, gap=3),
                                    (ps + 32, [(16, 2 * i * ps + 7) for i in range(6)], 12 * ps + 7)):
        surf = atlas(faces, rowbytes, origins[:n], rows, seed=rowbytes)[0]
        got = render_from_plan_with_layout(host, surf, rowbytes, origins, pm, bg, rubix)
        assert np.array_equal(got, want), (globe, lens, rowbytes, int((got != want).sum()))
