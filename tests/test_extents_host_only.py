"""The lensmap and the tile plan at the edges of their fields, without a GPU.

* Tile origins are 16-bit (TileDesc::px / py): a screen up to 65536 pixels wide or tall is planned and the plan,
  interpreted on the CPU the way the kernels read it, must reproduce the reference's render; a wider or taller
  screen gets no plan at all (the flat kernels serve it), rather than tiles whose origins wrapped onto the first
  tiles' pixels.
* Texel indices are 28-bit (BLINKY_LM_INDEX_MASK): plates up to 6688 texels are accepted, 6689 is refused, and at
  6688 the packed entries keep the index and the tint bits apart."""
import numpy as np
import pytest

from test_tile_plan import render_from_plan

LM_VALID, LM_INDEX_MASK, LM_TINT_SHIFT = 0x80000000, 0x0FFFFFFF, 28
MAX_PS = 6688          # largest plate size with 6 * ps^2 - 1 < 2^28


def _setup(host, globe, lens, zoom, rubix):
    host.command(f"f_globe {globe}")
    host.command(f"f_lens {lens}")
    host.command(zoom)
    host.set_rubix(rubix)


@pytest.mark.parametrize("w,h", [(65536, 8), (65537, 8), (65600, 8), (8, 65536), (8, 65537), (8, 65600)])
def test_tile_plan_across_the_65536_pixel_boundary(bb, host, restate, palette, w, h):
    ps = 16
    _setup(host, "cube", "equirect", "f_cover", True)
    host.build_lensmap(w, h, ps, threads=bb.usable_cpus())
    idx, tint = host.lensmap()
    om = restate.build("cube", "equirect", w, h, ps, zoom=("f_cover", 0))
    assert np.array_equal(idx, om["idx"]) and np.array_equal(tint, om["tint"])
    # f_cover maps the pixels past 65536 too: a wrapped tile origin would have real pixels to lose
    assert (idx[:, 65536:] >= 0).any() if w > 65536 else (idx[65536:, :] >= 0).any() if h > 65536 else (idx >= 0).all()
    tiles, entries = host.tile_plan()
    if max(w, h) > 65536:
        assert tiles.size == 0 and entries.size == 0, (w, h, tiles.size)
        assert host.plan_summary.startswith("tiles 0x0 "), host.plan_summary
        return
    assert tiles.size == ((w + 31) // 32) * ((h + 31) // 32)
    assert int(tiles["px"].max()) == (w - 1) // 32 * 32 and int(tiles["py"].max()) == (h - 1) // 32 * 32
    faces = bb.synthetic_faces(host.numplates, ps, 3)
    bg = bb.synthetic_background(w, h)
    pm = restate.palmaps(palette)
    want = restate.render(om["idx"], om["tint"], faces, pm, True, background=bg)
    got = render_from_plan(host, faces, pm, bg, True)
    assert np.array_equal(got, want), int((got != want).sum())


def _check_packed(host):
    """the packed entries decode to exactly lensmap()'s idx and tint"""
    idx, tint = host.lensmap()
    packed = host.lensmap_packed()
    valid = (packed & LM_VALID) != 0
    assert np.array_equal(valid, idx >= 0)
    assert np.array_equal(np.where(valid, packed & LM_INDEX_MASK, 0), np.where(valid, idx, 0).astype(np.uint32))
    ptint = (packed >> LM_TINT_SHIFT) & 7
    assert np.array_equal(ptint, np.where(tint == 255, 7, tint).astype(np.uint32))
    return idx, tint


def test_plate_size_at_the_28_bit_texel_index_limit(bb, host, restate, palette):
    w, h = 192, 96
    # equirect f_contain samples every plate, plate 5 included: indices of 5 * ps^2 and up set bits 26 and 27
    _setup(host, "cube", "equirect", "f_contain", True)
    host.build_lensmap(w, h, MAX_PS, threads=bb.usable_cpus())
    assert host.platesize == MAX_PS
    idx, tint = _check_packed(host)
    om = restate.build("cube", "equirect", w, h, MAX_PS, zoom=("f_contain", 0))
    assert np.array_equal(idx, om["idx"]) and np.array_equal(tint, om["tint"])
    assert int(idx.max()) >= 5 * MAX_PS * MAX_PS and int(idx.max()) < 6 * MAX_PS * MAX_PS <= LM_INDEX_MASK + 1
    assert set(np.unique(tint[idx >= 0]).tolist()) <= set(range(6)) | {255} and (tint[idx >= 0] < 6).any()
    faces = bb.synthetic_faces(6, MAX_PS, 1)
    pm = restate.palmaps(palette)
    bg = bb.synthetic_background(w, h)
    want = restate.render(om["idx"], om["tint"], faces, pm, True, background=bg)
    assert np.array_equal(render_from_plan(host, faces, pm, bg, True), want)

    with pytest.raises(bb.BlinkyError) as e:
        host.build_lensmap(w, h, MAX_PS + 1, threads=1)
    assert e.value.code == bb.E_INVALID and "28-bit texel index" in str(e.value)


# a narrow view into the far corner of the cube's bottom plate (5): magnified, so most tiles are BOX tiles, whose
# box origins (int16 TileDesc::box_x / box_y) lie more than 6000 texels into a 6688 plate
CORNER_ZOOM_LENS = """lens_width=0.02 lens_height=0.01 onload='f_contain'
function lens_inverse(x, y) return 0.9 + x, -1, -0.9 + y end"""


def test_box_tiles_deep_in_the_largest_plate(bb, host, restate, palette):
    w, h = 192, 96
    _setup(host, "cube", "equirect", "f_contain", True)
    host.load_lens("corner_zoom", CORNER_ZOOM_LENS)
    host.build_lensmap(w, h, MAX_PS, threads=2)
    idx, tint = _check_packed(host)
    assert (idx >= 5 * MAX_PS * MAX_PS).all()
    tiles, _ = host.tile_plan()
    is_box = np.isin(tiles["type"] & 3, (1, 3))
    assert is_box.mean() > 0.5 and int(tiles["box_x"][is_box].min()) > 6000 and int(tiles["box_y"][is_box].min()) > 6000
    # the plan interpreted on the CPU (box cut-outs from the plate) against render_lensmap of the same map
    faces = bb.synthetic_faces(6, MAX_PS, 2)
    pm = restate.palmaps(palette)
    bg = bb.synthetic_background(w, h)
    want = restate.render(idx, tint, faces, pm, True, background=bg)
    assert np.array_equal(render_from_plan(host, faces, pm, bg, True), want)


# the left half of the screen looks at the last texel of the cube's bottom plate (5; index 6 * 6688^2 - 1, on the
# rubix grid's padding: no tint), the right half into a rubix cell near that corner (tint 5)
CORNER_LENS = """lens_width=1 lens_height=1 onload='f_contain'
function lens_inverse(x, y)
  if x < 0 then return 0.9999, -1, -0.9999 end
  return 0.9, -1, -0.9
end"""


def test_largest_texel_index_leaves_the_tint_bits_alone(bb, host):
    _setup(host, "cube", "equirect", "f_contain", True)
    host.load_lens("corner", CORNER_LENS)
    host.build_lensmap(4, 4, MAX_PS, threads=1)
    idx, tint = _check_packed(host)
    packed = host.lensmap_packed()
    last = 6 * MAX_PS * MAX_PS - 1
    assert (idx[:, :2] == last).all() and (tint[:, :2] == 255).all()
    assert (packed[:, :2] == LM_VALID | 7 << LM_TINT_SHIFT | last).all()
    ps2 = MAX_PS * MAX_PS
    near = 5 * ps2 + int(0.95 * MAX_PS) * MAX_PS + int(0.95 * MAX_PS)
    assert (idx[:, 2:] == near).all() and (tint[:, 2:] == 5).all()
    assert (packed[:, 2:] == LM_VALID | 5 << LM_TINT_SHIFT | near).all()
