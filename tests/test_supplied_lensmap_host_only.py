"""Supplied lensmaps (blinky_set_lensmap) on host-only contexts: the caller's packed map replaces the lensmap as a
build would.  A build's own map fed back reproduces the build's state; refused maps change nothing; unmapped entries
normalise; the tile plan of random and adversarial maps, interpreted on the CPU the way tests/test_tile_plan.py
does, equals a direct gather of the map.  An independent planner written here pins the plan byte for byte, and
compiling make_tile_plan against altered copies of the shared per-tile functions (tile_plan.h) shows that it
catches them drifting.  The same maps go through the GPU planner in tests/test_gpu_supplied_lensmap.py."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_tile_plan import render_from_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VALID, TINT_NONE = 0x80000000, 7

# shipped lenses sampled for the round trip (the GPU file covers every lens)
SAMPLE_LENSES = [("panini", "f_fov 180"), ("stereographic", "f_fov 200"), ("hammer", "f_contain"), ("quincuncial", "f_cover"),
                 ("sinusoidal", "f_contain"), ("fisheye1", "f_contain")]   # sinusoidal: a forward-built map


def state(fe):
    """everything a supplied map must reproduce"""
    tiles, entries = fe.tile_plan()
    idx, tint = fe.lensmap()
    return {"idx": idx, "tint": tint, "packed": fe.lensmap_packed(), "display": fe.display(), "mapped": fe.mapped_pixels,
            "upload": fe.upload_bytes_per_frame, "tiles": tiles.tobytes(), "entries": entries.tobytes(), "digest": fe.plan_digest(),
            "size": (fe.width, fe.height, fe.platesize)}


def assert_same_state(a, b):
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert np.array_equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


# ---- maps -------------------------------------------------------------------------------------------------------

def pack(idx, tint, valid):
    return np.where(valid, VALID | (tint.astype(np.uint32) << 28) | idx.astype(np.uint32), TINT_NONE << 28).astype(np.uint32)


def shaped_map(rng, W, H, ps, nplates, shapes, tinted=True):
    """every tile maps onto one plate and spans a box of a shape drawn from `shapes` ((w, h) texels): many distinct
    box shapes, so the planner has to coarsen the box heights"""
    idx = np.zeros((H, W), np.int64)
    tint = np.full((H, W), TINT_NONE, np.int64)
    for y0 in range(0, H, 32):
        for x0 in range(0, W, 32):
            w, h = shapes[rng.integers(len(shapes))]
            bx = int(rng.integers(0, (ps - w) // 16 + 1)) * 16
            by = int(rng.integers(0, ps - h + 1))
            c = np.round(np.arange(32) * (w - 1) / 31).astype(np.int64)
            r = np.round(np.arange(32) * (h - 1) / 31).astype(np.int64)
            p = int(rng.integers(nplates))
            blk = p * ps * ps + (by + r[:, None]) * ps + bx + c[None, :]
            idx[y0:y0 + 32, x0:x0 + 32] = blk[:min(32, H - y0), :min(32, W - x0)]
            if tinted and rng.random() < 0.5:
                t = tint[y0:y0 + 32, x0:x0 + 32]
                t[rng.random(t.shape) < 0.5] = p % 6
    valid = rng.random((H, W)) < 0.97
    return pack(idx, tint, valid)


def box_shapes(max_box, heights):
    return [(w, h) for w in range(16, 257, 16) for h in heights if w * h <= max_box]


def random_map(kind, seed=0):
    """(packed [H, W], platesize, numplates, max_box) of one of the adversarial map kinds"""
    rng = np.random.default_rng(seed)
    if kind == "mixed":          # plates, tints and validity at random: seams everywhere, mostly GATHER tiles
        W, H, ps, n = 203, 117, 64, 6
        idx = rng.integers(0, n * ps * ps, (H, W))
        tint = rng.choice([0, 1, 2, 3, 4, 5, 7], (H, W))
        return pack(idx, tint, rng.random((H, W)) < 0.8), ps, n, 8192
    if kind == "seams":          # every tile straddles two plates
        W, H, ps, n = 160, 96, 64, 3
        y, x = np.mgrid[0:H, 0:W]
        plate = (x % 32 >= 16).astype(np.int64) + (y % 64 >= 32)
        idx = plate * ps * ps + (y % ps) * ps + x % ps
        return pack(idx, np.full((H, W), TINT_NONE), np.ones((H, W), bool)), ps, n, 8192
    if kind == "smooth":         # a coherent zoom of one plate per screen quadrant: BOX / BOX_FULL tiles, odd width
        W, H, ps, n = 333, 201, 128, 4
        y, x = np.mgrid[0:H, 0:W]
        plate = (x >= W // 2).astype(np.int64) + 2 * (y >= H // 2)
        px = (x * 0.37).astype(np.int64) % ps
        py = (y * 0.61).astype(np.int64) % ps
        tint = np.where((x // 40 + y // 40) % 3 == 0, plate, TINT_NONE)
        return pack(plate * ps * ps + py * ps + px, tint, (x - W / 2) ** 2 + (y - H / 2) ** 2 < (W / 2.2) ** 2), ps, n, 8192
    if kind == "ps-odd":         # platesize not a multiple of 16: GATHER tiles only
        W, H, ps, n = 150, 70, 100, 6
        y, x = np.mgrid[0:H, 0:W]
        idx = (x // 60) * ps * ps + (y % ps) * ps + x % ps
        return pack(idx, np.full((H, W), TINT_NONE), np.ones((H, W), bool)), ps, n, 8192
    if kind == "gran16":
        return shaped_map(rng, 640, 608, 512, 6, box_shapes(8192, range(8, 65, 8))), 512, 6, 8192
    if kind == "gran32":
        return shaped_map(rng, 736, 640, 512, 6, box_shapes(8192, range(8, 257, 8))), 512, 6, 8192
    if kind == "gran64":         # (BLINKY_MAX_BOX=16384)
        return shaped_map(rng, 736, 640, 512, 6, box_shapes(16384, range(8, 257, 8))), 512, 6, 16384
    raise ValueError(kind)


RANDOM_KINDS = ["mixed", "seams", "smooth", "ps-odd", "gran16", "gran32", "gran64"]
GRANULARITY = {"gran16": 16, "gran32": 32, "gran64": 64}


def plan_granularity(tiles):
    h = tiles["box_h8"][np.isin(tiles["type"] & 3, (1, 3))].astype(np.int64) * 8
    return max(g for g in (8, 16, 32, 64) if (h % g == 0).all())


def direct_gather(packed, faces, lut, bg, rubix):
    """the warp's definition: where(valid, lut[tint][faces[idx]], background)"""
    valid = (packed & VALID) != 0
    px = faces.reshape(-1)[np.where(valid, packed & 0x0FFFFFFF, 0).astype(np.int64)]
    if rubix:
        px = lut[((packed >> 28) & 7).astype(np.int64), px]
    return np.where(valid, px, bg)


def full_lut(palmaps):
    return np.concatenate([palmaps, np.arange(256, dtype=np.uint8)[None], np.arange(256, dtype=np.uint8)[None]])


# ---- an independent planner --------------------------------------------------------------------------------------

def py_plan(packed, ps, max_box=8192):
    """The tile plan of DESIGN.md section 3 written out directly: (tile descriptors, entry bytes)."""
    import blinky_b200 as bb

    H, W = packed.shape
    tx_n, ty_n = -(-W // 32), -(-H // 32)
    P = np.zeros((ty_n * 32, tx_n * 32), np.uint32)
    P[:H, :W] = packed
    ps2 = ps * ps
    lanes = np.arange(32)[:, None]
    i = np.arange(32)[None, :]
    lr, lc = (lanes >> 3) + 4 * (i >> 2), 4 * (lanes & 7) + (i & 3)
    for gran in (8, 16, 32, 64):
        tiles, shapes = [], []
        for ty in range(ty_n):
            for tx in range(tx_n):
                t = P[ty * 32:ty * 32 + 32, tx * 32:tx * 32 + 32].astype(np.int64)
                valid = (t >> 31) & 1 == 1
                d = {"px": tx * 32, "py": ty * 32, "box_x": 0, "box_y": 0, "plate": 0, "box_w16": 0, "box_h8": 0}
                if not valid.any():
                    tiles.append((2, 0, d, b""))
                    continue
                idx = t & 0x0FFFFFFF
                plate, rem = idx // ps2, idx % ps2
                py, px, tint = rem // ps, rem % ps, (t >> 28) & 7
                tinted = valid & (tint != 7)
                box = ps % 16 == 0 and len(np.unique(plate[valid])) == 1 and len(np.unique(tint[tinted])) <= 1
                if box:
                    minx = int(px[valid].min()) & ~15
                    miny = int(py[valid].min())
                    bw = -(-(int(px[valid].max()) - minx + 1) // 16) * 16
                    bh = -(-(int(py[valid].max()) - miny + 1) // gran) * gran
                    box = bw <= 256 and bh <= 256 and bw * bh <= max_box
                if not box:
                    tiles.append((1, 2, d, t.astype("<u4").tobytes()))
                    continue
                e16 = np.where(valid, 0x8000 | ((py - miny) * bw + (px - minx)), 0).astype("<u2")
                ent = np.zeros((4, 32, 8), "<u2")
                ent[i >> 3, lanes, i & 7] = e16[lr, lc]
                flags = (tinted[lr, lc].astype(np.uint64) << i.astype(np.uint64)).sum(axis=1).astype("<u4")
                tile_tint = int(tint[tinted][0]) if tinted.any() else 7
                d.update(box_x=minx, box_y=miny, plate=int(plate[valid][0]) | tile_tint << 3, box_w16=bw // 16, box_h8=bh // 8)
                shape = (bw // 16) << 8 | bh // 8
                if shape not in shapes:
                    shapes.append(shape)
                tiles.append((0, 3 if valid.all() else 1, d, ent.tobytes() + flags.tobytes()))
        if len(shapes) <= 64:
            break
    out = np.zeros(len(tiles), bb.Fisheye.TILE_DTYPE)
    entries = bytearray()
    n, shape_order = 0, []
    for cls in (0, 1, 2):
        for c, typ, d, blk in tiles:
            if c != cls:
                continue
            for k, v in d.items():
                out[n][k] = v
            out[n]["entry_offset"] = len(entries)
            if cls == 0:
                shape = d["box_w16"] << 8 | d["box_h8"]
                if shape not in shape_order:
                    shape_order.append(shape)
                typ |= shape_order.index(shape) << 2
            out[n]["type"] = typ
            entries += blk
            n += 1
    return out, np.frombuffer(bytes(entries) + bytes(16), np.uint8)


# ---- tests --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("globe", ["cube", "fast", "trism"])
@pytest.mark.parametrize("lens,zoom", SAMPLE_LENSES)
def test_a_builds_own_map_fed_back_reproduces_the_build(bb, palette, host, globe, lens, zoom):
    host.command(f"f_globe {globe}")
    host.command(f"f_lens {lens}")
    host.command(zoom)
    host.set_rubix(True)
    host.build_lensmap(200, 120, 64, threads=2)
    want = state(host)
    n = host.numplates
    other = bb.Fisheye(device=None, palette=palette)
    try:
        other.set_lensmap(want["packed"], 64, n)
        assert_same_state(want, state(other))
        assert "supplied (host memory)" in other.build_info
    finally:
        other.close()
    host.set_lensmap(want["packed"], 64, n)   # over the build itself: unchanged
    assert_same_state(want, state(host))


def test_unmapped_entries_with_junk_bits_normalise(host):
    rng = np.random.default_rng(3)
    H, W, ps = 50, 70, 32
    m = rng.integers(0, 2**31, (H, W), dtype=np.uint64).astype(np.uint32)   # bit 31 clear: all unmapped, any other bits
    m[::3, ::2] |= np.uint32(VALID)
    m[::3, ::2] &= np.uint32(0xF0000000 | 0x3FF)                            # valid: index < 6 * 32^2 = 6144
    m[::3, ::2] = np.where(((m[::3, ::2] >> 28) & 7) == 6, m[::3, ::2] | np.uint32(1 << 28), m[::3, ::2])   # no tint 6
    host.set_lensmap(m, ps, 6)
    valid = (m & VALID) != 0
    want = np.where(valid, m, np.uint32(TINT_NONE << 28))
    assert np.array_equal(host.lensmap_packed(), want)
    idx, tint = host.lensmap()
    assert (idx[~valid] == -1).all() and (tint[~valid] == 255).all()
    assert np.array_equal(idx[valid], (m[valid] & 0x0FFFFFFF).astype(np.int32))
    assert host.mapped_pixels == int(valid.sum())
    other_tiles, other_entries = py_plan(want, ps)
    tiles, entries = host.tile_plan()
    assert tiles.tobytes() == other_tiles.tobytes() and entries.tobytes() == other_entries.tobytes()


def refusals(ps=32, n=6, W=40, H=30):
    """(description, width, height, platesize, numplates, map) that must all be refused"""
    ok = np.full((H, W), TINT_NONE << 28, np.uint32)
    ok[5, 5] = VALID | 7 << 28 | 12

    def with_entry(e):
        m = ok.copy()
        m[7, 9] = e
        return m

    return [
        ("NULL map", W, H, ps, n, None),
        ("width 0", 0, H, ps, n, ok),
        ("height -1", W, -1, ps, n, ok),
        ("numplates 0", W, H, ps, 0, ok),
        ("numplates 7", W, H, ps, 7, ok),
        ("platesize 0", W, H, 0, n, ok),
        ("numplates * ps^2 above 2^28", W, H, 6689, 6, ok),
        ("index = numplates * ps^2", W, H, ps, n, with_entry(VALID | 7 << 28 | n * ps * ps)),
        ("index beyond the plates, a smaller numplates", W, H, ps, 2, with_entry(VALID | 7 << 28 | 2 * ps * ps + 5)),
        ("tint 6", W, H, ps, n, with_entry(VALID | 6 << 28 | 3)),
    ]


def set_raw(bb, fe, W, H, ps, n, m):
    ptr = None if m is None else np.ascontiguousarray(m).ctypes.data
    return bb.load_library().blinky_set_lensmap(fe._ctx, W, H, ps, n, ptr)


def test_refusals_change_nothing(bb, host):
    host.command("f_globe cube")
    host.command("f_lens stereographic")
    host.command("f_fov 200")
    host.build_lensmap(96, 64, 32)
    want = state(host)
    for what, W, H, ps, n, m in refusals():
        assert set_raw(bb, host, W, H, ps, n, m) == bb.E_INVALID, what
        assert bb.load_library().blinky_last_error(host._ctx).decode().startswith("blinky_set_lensmap"), what
        assert_same_state(want, state(host))
    # the largest plates are accepted: 6 * 6688^2 <= 2^28
    m = np.full((2, 3), TINT_NONE << 28, np.uint32)
    m[1, 2] = VALID | (6 * 6688 * 6688 - 1)
    host.set_lensmap(m, 6688, 6)
    assert host.lensmap()[0][1, 2] == 6 * 6688 * 6688 - 1


def test_needs_rebuild_follows_the_supplied_map(host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    m = np.full((48, 64), TINT_NONE << 28, np.uint32)
    m[10:20, 10:30] = VALID | 7 << 28 | 100
    assert host.needs_rebuild(64, 48, 32)
    host.set_lensmap(m, 32, 6)
    assert not host.needs_rebuild(64, 48, 32)
    assert host.needs_rebuild(64, 48, 0)          # 0: the reference's platesize, min(w, h) = 48
    assert host.needs_rebuild(65, 48, 32)
    host.command("f_fov 170")                     # a zoom change
    assert host.needs_rebuild(64, 48, 32)
    host.set_lensmap(m, 32, 6)
    assert not host.needs_rebuild(64, 48, 32)
    assert host.lens_name == "panini" and host.zoom_fov == 170 and host.globe_name == "cube"   # the settings stay
    host.command("f_lens hammer")                 # a lens change
    assert host.needs_rebuild(64, 48, 32)
    host.set_lensmap(m, 32, 6)
    host.command("f_globe trism")                 # a globe change
    assert host.needs_rebuild(64, 48, 32)
    assert host.display() == [1, 0, 0, 0, 0, 0]   # the map's plates, whatever the globe


@pytest.mark.parametrize("kind", RANDOM_KINDS)
def test_plan_of_random_maps_interpreted_on_the_cpu_equals_a_direct_gather(bb, host, restate, palette, monkeypatch, kind):
    m, ps, n, max_box = random_map(kind)
    if max_box != 8192:
        monkeypatch.setenv("BLINKY_MAX_BOX", str(max_box))
    host.command("f_globe cube")        # six plates of palette LUTs for the interpretation
    host.set_lensmap(m, ps, n)
    H, W = m.shape
    faces = np.random.default_rng(9).integers(0, 256, (6, ps, ps), dtype=np.uint8)
    bg = bb.synthetic_background(W, H)
    pm = restate.palmaps(palette)
    for rubix in (False, True):
        got = render_from_plan(host, faces, pm, bg, rubix, max_box=max_box)
        assert np.array_equal(got, direct_gather(m, faces, full_lut(pm), bg, rubix)), (kind, rubix)
    tiles, entries = host.tile_plan()
    want_tiles, want_entries = py_plan(m, ps, max_box)
    assert tiles.tobytes() == want_tiles.tobytes() and entries.tobytes() == want_entries.tobytes(), kind
    types = tiles["type"] & 3
    if kind in GRANULARITY:
        assert plan_granularity(tiles) == GRANULARITY[kind]
        assert len(np.unique(tiles["type"][np.isin(types, (1, 3))] >> 2)) <= 64
    if kind == "seams":
        assert (types == 2).all()
    if kind == "ps-odd":
        assert not np.isin(types, (1, 3)).any()
    if kind == "smooth":
        assert (types == 3).any() and (types == 1).any() and (types == 0).any()


# ---- the shared per-tile functions, pinned --------------------------------------------------------------------------

MUTATIONS = [
    ("box origin on 32 texels", "*box_x = minx & ~15u;", "*box_x = minx & ~31u;"),
    ("box height one granule too tall", "*bh = ((maxy - miny + 1) + g - 1) / g * g;", "*bh = ((maxy - miny + 1) + g - 1) / g * g + g;"),
    ("box entry row pitch", "((py - box_y) * bw + (px - box_x))", "((py - box_y) * (bw + 16) + (px - box_x))"),
    ("tint flag", "*tinted = ((e >> 28) & 7u) != 7u;", "*tinted = ((e >> 28) & 7u) != 6u;"),
    ("lane order", "return ((i >> 3) * 32 + lane) * 8 + (i & 7);", "return ((i >> 3) * 32 + lane) * 8 + (7 - (i & 7));"),
]

DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "tile_plan.h"
int main(int argc, char **argv) {
    const int W = atoi(argv[1]), H = atoi(argv[2]), ps = atoi(argv[3]);
    std::vector<uint32_t> m(static_cast<size_t>(W) * H);
    FILE *f = fopen(argv[4], "rb");
    if (fread(m.data(), 4, m.size(), f) != m.size()) return 2;
    fclose(f);
    blinky::TilePlan p = blinky::make_tile_plan(m.data(), W, H, ps, ps % 16 == 0, 1);
    f = fopen(argv[5], "wb");
    fwrite(p.tiles.data(), sizeof(blinky::TileDesc), p.tiles.size(), f);
    fclose(f);
    f = fopen(argv[6], "wb");
    fwrite(p.entries.data(), 1, p.entries.size(), f);
    fclose(f);
    return 0;
}
"""


def plan_with_header(tmp_path, header_text, m, ps):
    """make_tile_plan compiled against `header_text` as tile_plan.h, run on map m"""
    src = tmp_path / "blinky_b200" / "csrc"
    src.mkdir(parents=True, exist_ok=True)
    (tmp_path / "include").mkdir(exist_ok=True)
    shutil.copy(os.path.join(ROOT, "include", "blinky_b200.h"), tmp_path / "include")
    for f in ("tile_plan.cpp", "parallel.h"):
        shutil.copy(os.path.join(ROOT, "blinky_b200", "csrc", f), src)
    (src / "tile_plan.h").write_text(header_text)
    (src / "driver.cpp").write_text(DRIVER)
    exe = src / "plan"
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-pthread", "-I", str(src), str(src / "driver.cpp"), str(src / "tile_plan.cpp"), "-o", str(exe)],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:2000]
    H, W = m.shape
    (src / "map.bin").write_bytes(np.ascontiguousarray(m, "<u4").tobytes())
    r = subprocess.run([str(exe), str(W), str(H), str(ps), str(src / "map.bin"), str(src / "tiles.bin"), str(src / "entries.bin")],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    return (src / "tiles.bin").read_bytes(), (src / "entries.bin").read_bytes()


def test_the_shared_per_tile_functions_cannot_drift_unnoticed(bb, tmp_path):
    header = open(os.path.join(ROOT, "blinky_b200", "csrc", "tile_plan.h")).read()
    m, ps, _, _ = random_map("smooth", 4)
    want_tiles, want_entries = py_plan(m, ps)
    want = (want_tiles.tobytes(), want_entries.tobytes())
    assert plan_with_header(tmp_path / "same", header, m, ps) == want
    for what, old, new in MUTATIONS:
        assert header.count(old) == 1, what
        assert plan_with_header(tmp_path / what.replace(" ", "_"), header.replace(old, new), m, ps) != want, what
