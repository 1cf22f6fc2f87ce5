"""Every instance of the four warp kernels, checked byte for byte against the CPU oracle, on the GPU.

The ring kernel, K3 (warp_tile_gather_kernel), K1 (warp_gather_kernel) and K0 (warp_scalar_kernel) each have one
instance per combination of the flags RUBIX x RGBA x KEEP x TABLES x LAYOUT, with TABLES only in RGBA: 24 variants.
For each variant the test warps four lensmaps (globes of 4, 6, 5 and 2 plates) into random-filled screens, from dense
faces or, for the layout variants, from three face layouts, with each placement forced in turn: the ring kernel with
its gather CTAs, K3 in front of it, K1 and K0.  Every byte of the output buffer is compared with expected_screen, which
is built from the oracle's 8-bit frames alone.  last_kernel tells which instances ran; each variant's test asserts that
all five of its cells (four kernels, plus the gather CTAs of the ring kernel's launch) were checked.  The CPU suite
pins expected_screen to the compiled reference's frames, and pins VARIANTS and KERNELS to the instances the built
library holds (test_variant_matrix_host_only.py)."""
import re
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KERNELS = ("warp_ring_kernel", "warp_tile_gather_kernel", "warp_gather_kernel", "warp_scalar_kernel")
GATHER_CTAS = "gather CTAs"   # the ledger's name for the ring kernel's gather_item path
FLAGS = ("rubix", "rgba", "keep", "tables", "layout")   # the kernels' template arguments, in order

# (rubix, rgba, keep, tables, layout) of every instance: per-frame tables exist only in RGBA
VARIANTS = [v for v in ((i & 1, i >> 1 & 1, i >> 2 & 1, i >> 3 & 1, i >> 4 & 1) for i in range(32)) if v[1] or not v[3]]


def variant_name(v) -> str:
    """the variant as last_kernel spells it: rubix= and rgba= with their values, then the flags that are set"""
    rubix, rgba, keep, tables, layout = v
    return f"rubix={rubix},rgba={rgba}" + "".join(f",{f}=1" for f, on in zip(FLAGS[2:], v[2:]) if on)


def expected_screen(fill, want8, idx, *, nframes, x0, y0, rowbytes, frame_stride, keep, table=None, tables=None):
    """The bytes a warp must leave in a flat output buffer that held `fill`: frame f's view rectangle, at pixel (x0, y0)
    of a screen with `rowbytes` bytes per row, frame_stride bytes after frame f-1's, holds want8[f] (8-bit),
    table[want8[f]] (RGBA, uint32 table) or tables[f][want8[f]] (per-frame tables); with keep only the pixels where
    idx >= 0.  Every other byte keeps its fill."""
    H, W = idx.shape
    rgba = table is not None or tables is not None
    bpp = 4 if rgba else 1
    out = np.array(fill, np.uint8, copy=True).reshape(-1)
    mask = np.repeat(idx >= 0, bpp, axis=1)
    for f in range(nframes):
        px = want8[f]
        if rgba:
            px = np.ascontiguousarray((tables[f] if tables is not None else table)[px], dtype="<u4").view(np.uint8).reshape(H, W * 4)
        start = f * frame_stride + y0 * rowbytes
        rect = out[start:start + H * rowbytes].reshape(H, rowbytes)[:, x0 * bpp:(x0 + W) * bpp]
        if keep:
            rect[mask] = px[mask]
        else:
            rect[:] = px
    return out


# ---- what ran, from last_kernel ----------------------------------------------------------------------------------

LAUNCH = re.compile(r"(warp_ring_kernel|warp_tile_gather_kernel|warp_gather_kernel|warp_scalar_kernel)<([^>]*)> grid=(?:(\d+)\+(\d+))?")


def launches(last_kernel: str):
    """[(kernel, variant as last_kernel spells it, gather CTAs of a ring launch or None)]"""
    return [(m.group(1), m.group(2), int(m.group(4)) if m.group(4) else None) for m in LAUNCH.finditer(last_kernel)]


def cells_of(last_kernel: str) -> set:
    """the ledger's cells a warp exercised: (kernel, variant), and (GATHER_CTAS, variant) when gather CTAs rode along"""
    cells = set()
    for kernel, variant, extra in launches(last_kernel):
        cells.add((kernel, variant))
        if extra:
            cells.add((GATHER_CTAS, variant))
    return cells


# ---- lensmaps, faces, layouts ------------------------------------------------------------------------------------

MAPS = {
    # name: (globe, lens, zoom, (W, H, platesize))
    "tetra-hammer": ("tetra", "hammer", "f_contain", (400, 226, 192)),        # EMPTY, BOX, GATHER and BOX_FULL tiles; W, H % 32 != 0
    "cube-quincuncial": ("cube", "quincuncial", "f_cover", (320, 200, 256)),  # large boxes
    "trism-hammer": ("trism", "hammer", "f_contain", (236, 138, 96)),         # five plates
    "fast-panini": ("fast", "panini", "f_fov 160", (240, 136, 128)),          # two plates
}
NFRAMES = 17   # the most frames a warp here takes: K3's four-frame groups and the 3-frame units both end in a partial one
FCHUNK = "3"   # frames per ring unit (BLINKY_FCHUNK): 5 and 17 frames end in a partial unit


def layouts(ps, n):
    """name -> (rowbytes, origins of plates 0..n-1, rows) of the three face layouts"""
    atlas = [(c * (ps + 16), r * (ps + 16)) for r in range(2) for c in range(3)]
    padded = [(c * (ps + 32), 8 + r * (ps + 24)) for r in range(2) for c in range(3)]
    odd = [(c * (ps + 5) + 3, r * (ps + 7) + 1) for r in range(2) for c in range(3)]
    return {
        # rowbytes and every x a multiple of 16: the ring kernel takes it
        "aligned-atlas": (3 * (ps + 16), atlas[:n], 2 * ps + 16),
        # plate 0 in the last slot, padded rows and 5 extra rows: a kernel that ignores an origin, or takes plate i's
        # origin for plate j, reads other bytes
        "permuted-atlas": (3 * (ps + 32) + 48, [padded[n - 1]] + padded[:n - 1], 8 + 2 * (ps + 24) + 5),
        # x % 16 != 0: K1 (K0 for a ragged view)
        "odd-origins": (-(-(3 * ps + 13) // 16) * 16, odd[:n], 2 * ps + 8),
    }


def surfaces(faces, rowbytes, origins, rows, seed):
    """[N, rows, rowbytes] random bytes with plate i of each frame at origins[i]"""
    n, p, ps, _ = faces.shape
    out = np.random.default_rng(seed).integers(0, 256, (n, rows, rowbytes), dtype=np.uint8)
    for i in range(p):
        x, y = origins[i]
        out[:, y:y + ps, x:x + ps] = faces[:, i]
    return out


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch

    return torch


@pytest.fixture(scope="module")
def globes(bb, restate, palette, torch_mod, cuda_device):
    """name -> the context of one lensmap of MAPS and what its warps need: the map, the tile plan's counts, 17 frames of
    faces (dense and in each layout) and the oracle's 8-bit frames of them with rubix off and on"""
    torch = torch_mod
    pm = restate.palmaps(palette)
    out = {}
    try:
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("BLINKY_FCHUNK", FCHUNK)   # read when a context is created
            for k, (name, (globe, lens, zoom, (W, H, ps))) in enumerate(MAPS.items()):
                fe = bb.Fisheye(device=cuda_device, palette=palette)
                out[name] = g = types.SimpleNamespace(fe=fe)
                fe.command(f"f_globe {globe}")
                fe.command(f"f_lens {lens}")
                fe.command(zoom)
                fe.build_lensmap(W, H, ps, 8)
                n = fe.numplates
                bg = bb.synthetic_background(W, H)
                fe.set_background(bg)
                g.idx, tint = fe.lensmap()
                tiles = fe.tile_plan()[0]
                g.types = {int(t): int((tiles["type"] & 3 == t).sum()) for t in range(4)}
                faces = np.stack([bb.synthetic_faces(n, ps, 100 * k + f) for f in range(NFRAMES)])
                g.want8 = {r: np.stack([restate.render(g.idx, tint, faces[f], pm, bool(r), background=bg) for f in range(NFRAMES)])
                           for r in (0, 1)}
                g.faces = {"dense": (None, torch.from_numpy(faces).cuda())}
                for j, (lname, (rowbytes, origins, rows)) in enumerate(layouts(ps, n).items()):
                    surf = surfaces(faces, rowbytes, origins, rows, seed=10 * k + j)
                    g.faces[lname] = ((rowbytes, origins), torch.from_numpy(surf).cuda())
    except BaseException:
        for g in out.values():
            g.fe.close()
        raise
    assert all(out["tetra-hammer"].types.values()), out["tetra-hammer"].types   # all four tile types
    yield out
    for g in out.values():
        g.fe.close()


@pytest.fixture(scope="module")
def palettes(torch_mod):
    """(RGBA table, per-frame tables on the host [17, 256], the same on the device with a stride of 1024 + 48 bytes and
    0xdeadbeef in the 12 padding words of each)"""
    torch = torch_mod
    table = np.random.default_rng(5).integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32)
    tables = np.random.default_rng(6).integers(0, 2**32, (NFRAMES, 256), dtype=np.uint64).astype(np.uint32)
    padded = np.full((NFRAMES, 256 + 12), 0xdeadbeef, np.uint32)
    padded[:, :256] = tables
    d_padded = torch.from_numpy(padded.view(np.int32)).cuda()
    return table, tables, d_padded[:, :256]


# ---- the matrix --------------------------------------------------------------------------------------------------

# (name, frames, x0 of the view, blinky_set_kernel): the view is aligned to 16 bytes unless x0 is odd
PLACEMENTS = [
    ("ring", 1, 8, 0),      # GATHER tiles ride along as gather CTAs
    ("ring", 5, 8, 0),      # ... in two groups of frames, the second partial
    ("k3+ring", 17, 8, 0),  # > 8 frames: K3 in front of the ring kernel
    ("k1", 5, 8, 1),        # BLINKY_KERNEL_GATHER
    ("k0", 5, 3, 0),        # a view at an odd x0
]


def placement_kernels(placement, nframes, layout, g):
    """the kernels last_kernel must name: a face layout with odd x origins sends the ring kernel's warps to K1"""
    if placement == "k0":
        return {"warp_scalar_kernel"}
    if placement == "k1" or layout == "odd-origins":
        return {"warp_gather_kernel"}
    return {"warp_ring_kernel"} | ({"warp_tile_gather_kernel"} if g.types[2] and nframes > 8 else set())


def warp_and_check(torch, g, d_faces, variant, palettes, *, nframes, x0, seed, what):
    """One warp of `variant` into a random-filled flat buffer of screens (the view at (x0, 2), 3 guard rows below it,
    padding between frames), every byte compared with expected_screen.  Returns last_kernel."""
    rubix, rgba, keep, tables, _ = variant
    fe = g.fe
    H, W = g.idx.shape
    bpp = 4 if rgba else 1
    y0 = 2
    rowbytes = -(-(x0 + W + 13) * bpp // 16) * 16
    frame_stride = (y0 + H + 3) * rowbytes + 16 * bpp
    fill = np.random.default_rng(seed).integers(0, 256, nframes * frame_stride, dtype=np.uint8)
    d_screen = torch.from_numpy(fill).cuda()
    table, host_tables, d_tables = palettes
    fe.warp_view(d_faces, d_screen.data_ptr(), x0=x0, y0=y0, rowbytes=rowbytes, nframes=nframes, keep_unmapped=bool(keep),
                 rgba=bool(rgba), screen_stride=frame_stride, stream=torch.cuda.current_stream().cuda_stream,
                 tables=d_tables if tables else None)
    torch.cuda.synchronize()
    got = d_screen.cpu().numpy()
    want = expected_screen(fill, g.want8[rubix], g.idx, nframes=nframes, x0=x0, y0=y0, rowbytes=rowbytes,
                           frame_stride=frame_stride, keep=keep, table=table if rgba and not tables else None,
                           tables=host_tables if tables else None)
    if not np.array_equal(got, want):
        bad = np.flatnonzero(got != want)
        frames = sorted(set((bad // frame_stride).tolist()))
        pytest.fail(f"{what}: {bad.size} wrong bytes in frames {frames} — {fe.last_kernel}")
    return fe.last_kernel


@pytest.mark.parametrize("variant", VARIANTS, ids=variant_name)
def test_variant_against_the_oracle(globes, palettes, torch_mod, variant):
    torch = torch_mod
    rubix, rgba, keep, tables, layout = variant
    name = variant_name(variant)
    checked = set()
    seed = 0
    for gname, g in globes.items():
        fe = g.fe
        fe.set_rubix(bool(rubix))
        fe.set_rgba_table(palettes[0])
        for lname, (lay, d_faces) in g.faces.items():
            if (lname == "dense") == bool(layout):
                continue
            if lay:
                fe.set_face_layout(*lay)
            else:
                fe.set_face_layout()
            for placement, nframes, x0, kernel in PLACEMENTS:
                seed += 1
                what = f"{name} {gname} {lname} {placement} {nframes} frames"
                fe.set_kernel(kernel)
                try:
                    k = warp_and_check(torch, g, d_faces, variant, palettes, nframes=nframes, x0=x0, seed=seed, what=what)
                finally:
                    fe.set_kernel(0)
                ran = launches(k)
                assert {r[0] for r in ran} == placement_kernels(placement, nframes, lname, g), (what, k)
                assert all(v == name for _, v, _ in ran), (what, k)   # rubix=, rgba= and exactly the variant's flags
                if placement == "ring" and lname != "odd-origins":
                    assert (ran[0][2] > 0) == bool(g.types[2]), (what, k)   # gather CTAs exactly when there are GATHER tiles
                checked |= cells_of(k)
        fe.set_face_layout()
    missing = {(k, name) for k in KERNELS + (GATHER_CTAS,)} - checked
    assert not missing, f"{name}: never checked byte for byte: {sorted(c[0] for c in missing)}"
