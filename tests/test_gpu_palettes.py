"""Per-frame palette tables (blinky_warp_device_view_rgba_tables, the tables= argument of Fisheye.warp_view and
Fisheye.warp), on the GPU.

Frame f of a batch is expanded through its own 256-entry table, read from device memory when the launch runs.  Every
check compares every byte of the screens, guard rows and padding included, with the CPU oracle's 8-bit frame mapped
through tables[f]; the tables are seeded, random and distinct per frame, so a frame expanded through a neighbour's
table shows."""
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch

    return torch


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


def setup(fe, globe, lens, w, h, ps, zoom=None, rubix=False):
    fe.command(f"f_globe {globe}")
    fe.command(f"f_lens {lens}")
    if zoom:
        fe.command(zoom)
    fe.set_rubix(rubix)
    fe.build_lensmap(w, h, ps, 8)


def stream_of(torch):
    return torch.cuda.current_stream().cuda_stream


def random_tables(n, seed):
    return np.random.default_rng(seed).integers(0, 2**32, (n, 256), dtype=np.uint64).astype(np.uint32)


def device_tables(torch, tables, pad_words=0):
    """tables [N, 256] on the device with rows of 256 + pad_words words (stride (256 + pad_words) * 4 bytes)"""
    rows = np.zeros((len(tables), 256 + pad_words), np.uint32)
    rows[:, :256] = tables
    rows[:, 256:] = 0xdeadbeef   # padding a kernel must never read as a table entry
    return torch.from_numpy(rows.view(np.int32)).cuda()[:, :256]


def oracle_frames(bb, restate, palette, fe, faces, rubix, bg=None):
    idx, tint = fe.lensmap()
    pm = restate.palmaps(palette)
    return np.stack([restate.render(idx, tint, faces[i], pm, rubix, background=bg) for i in range(len(faces))])


def warp_into_screen(torch, fe, d_faces, want8, mapped, *, nframes, x0, y0, rowbytes, rows_below, pad, keep, tables,
                     d_tables, seed=0):
    """Warps `nframes` RGBA frames with per-frame tables into a random-filled flat device buffer of screens
    (rows_below guard rows under the rectangle, `pad` bytes between screens) and checks every byte of it against
    want8[f] mapped through tables[f].  Returns the kernel that ran."""
    W, H = fe.width, fe.height
    fstride = (y0 + H + rows_below) * rowbytes + pad
    fill = np.random.default_rng(seed).integers(0, 256, nframes * fstride, dtype=np.uint8)
    d_screen = torch.from_numpy(fill).cuda()
    fe.warp_view(d_faces, d_screen.data_ptr(), x0=x0, y0=y0, rowbytes=rowbytes, nframes=nframes, keep_unmapped=keep,
                 rgba=True, screen_stride=fstride, stream=stream_of(torch), tables=d_tables)
    torch.cuda.synchronize()
    got = d_screen.cpu().numpy()
    expect = fill.copy()
    mask = np.repeat(mapped, 4, axis=1)
    for f in range(nframes):
        start = f * fstride + y0 * rowbytes
        rect = expect[start:start + H * rowbytes].reshape(H, rowbytes)[:, x0 * 4:(x0 + W) * 4]
        px = tables[f][want8[f]].view(np.uint8).reshape(H, W * 4)
        if keep:
            rect[mask] = px[mask]
        else:
            rect[:] = px
    assert np.array_equal(got, expect), (fe.last_kernel, nframes, x0, y0, rowbytes, keep)
    return fe.last_kernel


# ---- oracle sweep ------------------------------------------------------------------------------------------------

SWEEP = {
    "panini-rubix": ("cube", "panini", None, (320, 200, 128), True),
    "hammer-contain-rubix": ("tetra", "hammer", "f_contain", (400, 226, 192), True),   # BOX, GATHER and EMPTY tiles
    "quincuncial-cover": ("cube", "quincuncial", "f_cover", (320, 200, 256), False),   # large boxes
    "fisheye1-ragged": ("cube", "fisheye1", None, (322, 150, 96), True),               # W % 4 != 0
}


def views(W):
    """RGBA (name, x0, y0, rowbytes, pad): an aligned view, an origin that is not 4-aligned, a pitch that is not 4
    pixels"""
    aligned = -(-(8 + W + 13) * 4 // 16) * 16
    return [("aligned", 8, 2, aligned, 64),
            ("odd-origin", 3, 1, aligned, 28),
            ("odd-pitch", 8, 2, (8 + W + 3) * 4, 28)]


@pytest.mark.parametrize("case", list(SWEEP))
def test_tables_against_oracle(bb, fe, restate, palette, torch_mod, case):
    """1, 5, 16 and 17 frames; keep on and off; aligned, odd-origin and odd-pitch views; kernel variants 0 and 1;
    table strides of 1024 and 1024 + 48 bytes.  Asserts which kernel ran: the ring kernel with GATHER tiles as extra
    CTAs of its launch (<= 8 frames) or behind the gather kernel (> 8 frames), the flat kernel, the per-pixel kernel."""
    torch = torch_mod
    globe, lens, zoom, (W, H, PS), rubix = SWEEP[case]
    setup(fe, globe, lens, W, H, PS, zoom, rubix)
    bg = bb.synthetic_background(W, H)
    fe.set_background(bg)
    fe.set_rgba_table(random_tables(1, 99)[0])   # the context's table: must not be the one used
    ngather = int(np.count_nonzero((fe.tile_plan()[0]["type"] & 3) == 2))
    if case.startswith("hammer"):
        assert ngather > 0
    idx, _ = fe.lensmap()
    mapped = idx >= 0
    N = 17
    faces = np.stack([bb.synthetic_faces(fe.numplates, PS, 50 + i) for i in range(N)])
    want8 = oracle_frames(bb, restate, palette, fe, faces, rubix, bg)
    d_faces = torch.from_numpy(faces).cuda()
    tables = random_tables(N, 7)
    seen = set()
    seed = 0
    for pad_words in (0, 12):
        d_tables = device_tables(torch, tables, pad_words)
        assert d_tables.stride(0) * 4 == 1024 + 4 * pad_words
        for kernel_variant in (0, 1):
            fe.set_kernel(kernel_variant)
            for nframes in (1, 5, 16, 17):
                for name, x0, y0, rowbytes, pad in views(W):
                    for keep in (False, True):
                        seed += 1
                        kernel = warp_into_screen(torch, fe, d_faces, want8, mapped, nframes=nframes, x0=x0, y0=y0,
                                                  rowbytes=rowbytes, rows_below=3, pad=pad, keep=keep, tables=tables,
                                                  d_tables=d_tables, seed=seed)
                        assert "tables=1" in kernel and ("keep=1" in kernel) == keep, kernel
                        vec = name == "aligned" and W % 4 == 0
                        if not vec:
                            assert "warp_scalar_kernel" in kernel, (case, name, kernel)
                        elif kernel_variant == 1:
                            assert "warp_gather_kernel" in kernel, (case, name, kernel)
                        else:
                            assert "warp_ring_kernel" in kernel, (case, name, kernel)
                            extra = int(re.search(r"grid=\d+\+(\d+)", kernel).group(1))
                            if ngather and nframes <= 8:
                                assert extra > 0 and "warp_tile_gather_kernel" not in kernel, kernel
                                seen.add("ring+gather CTAs")
                            elif ngather:
                                assert "warp_tile_gather_kernel" in kernel and extra == 0, kernel
                                seen.add("K3 + ring")
    fe.set_kernel(0)
    if ngather and W % 4 == 0:
        assert seen == {"ring+gather CTAs", "K3 + ring"}, seen


# ---- ring geometries ------------------------------------------------------------------------------------------------

RING_KNOBS = [
    {"BLINKY_RING_CTAS": "2", "BLINKY_STATIC_PCT": "0"},     # few warps, every unit from the ticket counter
    {"BLINKY_RING_CTAS": "16", "BLINKY_STATIC_PCT": "100"},  # as many warps as the registers allow, no tickets
    {"BLINKY_RING_BYTES": "128", "BLINKY_RING_BOXES": "6"},  # the smallest ring the plan allows: wraps all the time
    {"BLINKY_RING_BYTES": "32768", "BLINKY_RING_BOXES": "6", "BLINKY_RING_CTAS": "4"},  # a deep ring
    {"BLINKY_FCHUNK": "1"}, {"BLINKY_FCHUNK": "3"}, {"BLINKY_FCHUNK": "16"},             # unit = 1 / 3 / 16 frames
]


@pytest.mark.parametrize("knobs", RING_KNOBS, ids=lambda k: ",".join(f"{a[7:]}={b}" for a, b in k.items()))
def test_tables_ring_geometries(bb, restate, palette, torch_mod, cuda_device, knobs, monkeypatch):
    """The ring kernel restages its table slot once per frame, loading the next frame's table a frame ahead: the
    next frame moves across unit boundaries, tickets and ring wraps with the knobs.  Two plans (BOX, GATHER and EMPTY
    tiles with the rubix overlay; large boxes), 5 and 17 frames, dense and with keep_unmapped, against the oracle."""
    torch = torch_mod
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    for globe, lens, zoom, (W, H, PS), rubix in (("tetra", "hammer", "f_contain", (1000, 562, 512), True),
                                                 ("cube", "quincuncial", "f_cover", (1280, 720, 1024), False)):
        with bb.Fisheye(device=cuda_device, palette=palette) as f:   # the knobs are read when the context is created
            setup(f, globe, lens, W, H, PS, zoom, rubix)
            bg = bb.synthetic_background(W, H)
            f.set_background(bg)
            idx, _ = f.lensmap()
            N = 17
            faces = np.stack([bb.synthetic_faces(f.numplates, PS, 40 + i) for i in range(N)])
            want8 = oracle_frames(bb, restate, palette, f, faces, rubix, bg)
            d_faces = torch.from_numpy(faces).cuda()
            tables = random_tables(N, 11)
            d_tables = device_tables(torch, tables)
            for nframes in (5, 17):
                out = torch.zeros((nframes, H, W), dtype=torch.int32, device="cuda")
                f.warp(d_faces, out, nframes=nframes, rgba=True, stream=stream_of(torch), tables=d_tables)
                torch.cuda.synchronize()
                assert "warp_ring_kernel" in f.last_kernel and "tables=1" in f.last_kernel, f.last_kernel
                got = out.cpu().numpy().view(np.uint32)
                for i in range(nframes):
                    assert np.array_equal(got[i], tables[i][want8[i]]), (knobs, lens, nframes, i, f.last_kernel)
                kernel = warp_into_screen(torch, f, d_faces, want8, idx >= 0, nframes=nframes, x0=4, y0=3,
                                          rowbytes=(W + 16) * 4, rows_below=2, pad=64, keep=True, tables=tables,
                                          d_tables=d_tables, seed=nframes)
                assert "warp_ring_kernel" in kernel and "keep=1,tables=1" in kernel, kernel


# ---- equivalences ---------------------------------------------------------------------------------------------------

HAMMER = ("tetra", "hammer", "f_contain", (400, 226, 192), True)


def test_stride_zero_is_the_context_table(bb, fe, torch_mod):
    """One table at stride 0 gives what blinky_warp_device_view_rgba gives after set_rgba_table of the same table,
    through the same kernel instance; N copies of it at stride 1024 give the same bytes again."""
    torch = torch_mod
    globe, lens, zoom, (W, H, PS), rubix = HAMMER
    setup(fe, globe, lens, W, H, PS, zoom, rubix)
    fe.set_background(bb.synthetic_background(W, H))
    table = random_tables(1, 21)[0]
    fe.set_rgba_table(table)
    N = 16
    d_faces = torch.from_numpy(np.stack([bb.synthetic_faces(fe.numplates, PS, i) for i in range(N)])).cuda()
    one = torch.from_numpy(table.view(np.int32)).cuda()
    copies = device_tables(torch, np.repeat(table[None], N, axis=0))
    for kernel_variant in (0, 1):
        fe.set_kernel(kernel_variant)
        for nframes in (1, 5, N):
            for keep in (False, True):
                outs, kernels = [], []
                for tables in (None, one, copies):
                    out = torch.full((nframes, H + 2, W + 8), 7, dtype=torch.int32, device="cuda")
                    fe.warp_view(d_faces, out, x0=4, y0=1, nframes=nframes, keep_unmapped=keep, rgba=True,
                                 stream=stream_of(torch), tables=tables)
                    outs.append(out)
                    kernels.append(fe.last_kernel)
                torch.cuda.synchronize()
                assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), (kernel_variant, nframes, keep)
                assert kernels[0] == kernels[1], kernels
                assert "tables=1" not in kernels[1] and "tables=1" in kernels[2], kernels
    fe.set_kernel(0)


def test_plain_rgba_call_keeps_the_context_table(bb, fe, torch_mod):
    """A tables call neither reads nor changes the context's table: a plain RGBA warp after it still expands through
    the set_rgba_table table."""
    torch = torch_mod
    globe, lens, zoom, (W, H, PS), rubix = HAMMER
    setup(fe, globe, lens, W, H, PS, zoom, rubix)
    table = random_tables(1, 31)[0]
    fe.set_rgba_table(table)
    N = 5
    d_faces = torch.from_numpy(np.stack([bb.synthetic_faces(fe.numplates, PS, i) for i in range(N)])).cuda()
    ref = torch.zeros((N, H, W), dtype=torch.int32, device="cuda")
    fe.warp(d_faces, ref, nframes=N, rgba=True, stream=stream_of(torch))
    other = torch.zeros_like(ref)
    fe.warp(d_faces, other, nframes=N, rgba=True, stream=stream_of(torch),
            tables=device_tables(torch, random_tables(N, 32)))
    after = torch.zeros_like(ref)
    fe.warp(d_faces, after, nframes=N, rgba=True, stream=stream_of(torch))
    torch.cuda.synchronize()
    assert not torch.equal(ref, other)
    assert torch.equal(ref, after)
    assert "tables=1" not in fe.last_kernel


# ---- stream order and capture -----------------------------------------------------------------------------------------

def pinned(torch, tables):
    return torch.from_numpy(np.ascontiguousarray(tables).view(np.int32)).pin_memory()


def test_stream_order(bb, fe, restate, palette, torch_mod):
    """On one stream and with no synchronise in between: copy table A in, warp, copy table B in, warp.  The first
    warp uses A and the second B (1 frame, and 16 frames with a table each)."""
    torch = torch_mod
    globe, lens, zoom, (W, H, PS), rubix = HAMMER
    setup(fe, globe, lens, W, H, PS, zoom, rubix)
    bg = bb.synthetic_background(W, H)
    fe.set_background(bg)
    for nframes in (1, 16):
        faces = np.stack([bb.synthetic_faces(fe.numplates, PS, 60 + i) for i in range(nframes)])
        want8 = oracle_frames(bb, restate, palette, fe, faces, rubix, bg)
        d_faces = torch.from_numpy(faces).cuda()
        a, b = random_tables(nframes, 41), random_tables(nframes, 42)
        ha, hb = pinned(torch, a), pinned(torch, b)
        d_tables = torch.zeros((nframes, 256), dtype=torch.int32, device="cuda")
        outs = [torch.zeros((nframes, H, W), dtype=torch.int32, device="cuda") for _ in range(2)]
        torch.cuda.synchronize()
        d_tables.copy_(ha, non_blocking=True)
        fe.warp(d_faces, outs[0], nframes=nframes, rgba=True, stream=stream_of(torch), tables=d_tables)
        d_tables.copy_(hb, non_blocking=True)
        fe.warp(d_faces, outs[1], nframes=nframes, rgba=True, stream=stream_of(torch), tables=d_tables)
        torch.cuda.synchronize()
        for out, t in zip(outs, (a, b)):
            got = out.cpu().numpy().view(np.uint32)
            for i in range(nframes):
                assert np.array_equal(got[i], t[i][want8[i]]), (nframes, i)


def test_capture_reads_tables_at_replay(bb, fe, torch_mod):
    """A one-frame tables warp captured once and replayed three times, a new table copied in on the stream before each
    replay: each replay equals the eager warp with that table.  A captured 16-frame warp replays equal to eager."""
    torch = torch_mod
    globe, lens, zoom, (W, H, PS), rubix = HAMMER
    setup(fe, globe, lens, W, H, PS, zoom, rubix)
    fe.set_background(bb.synthetic_background(W, H))
    for nframes in (1, 16):
        d_faces = torch.from_numpy(np.stack([bb.synthetic_faces(fe.numplates, PS, 80 + i) for i in range(nframes)])).cuda()
        d_tables = device_tables(torch, random_tables(nframes, 50))
        out = torch.zeros((nframes, H + 4, W + 12), dtype=torch.int32, device="cuda")

        def warp(dst):
            fe.warp_view(d_faces, dst, x0=8, y0=2, nframes=nframes, rgba=True, tables=d_tables)

        warp(out)   # (eager first, as a host would)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            warp(out)
        assert "warp_ring_kernel" in fe.last_kernel and "tables=1" in fe.last_kernel, fe.last_kernel
        for r in range(3):
            host = pinned(torch, random_tables(nframes, 51 + r))
            out.zero_()
            d_tables.copy_(host, non_blocking=True)
            g.replay()
            want = torch.zeros_like(out)
            warp(want)
            torch.cuda.synchronize()
            assert torch.equal(out, want), (nframes, r)
            assert torch.equal(d_tables.cpu(), host), (nframes, r)
        del g
    fe.release_captures()


# ---- argument errors --------------------------------------------------------------------------------------------

def test_tables_argument_errors_launch_nothing(bb, fe, torch_mod):
    torch = torch_mod
    W, H, PS = 128, 96, 48
    setup(fe, "cube", "panini", W, H, PS)
    d_faces = torch.from_numpy(np.stack([bb.synthetic_faces(6, PS, i) for i in range(2)])).cuda()
    screen = torch.zeros(2 * 120 * 640 + 64, dtype=torch.uint8, device="cuda")
    tables = torch.zeros(4 * 512 + 16, dtype=torch.int32, device="cuda")
    base, tab = screen.data_ptr(), tables.data_ptr()
    lib = fe._lib
    ok = dict(faces=d_faces.data_ptr(), face_stride=6 * PS * PS, screen=base, stride=120 * 640, rowbytes=640, x0=8,
              y0=6, nframes=2, keep=0, tables=tab, table_stride=2048)

    def call(a):
        return lib.blinky_warp_device_view_rgba_tables(fe._ctx, a["faces"], a["face_stride"], a["screen"], a["stride"],
                                                       a["rowbytes"], a["x0"], a["y0"], a["nframes"], a["keep"],
                                                       a["tables"], a["table_stride"], stream_of(torch))

    bad = [
        ("NULL faces", {"faces": None}),
        ("NULL screen", {"screen": None}),
        ("x0 < 0", {"x0": -1}),
        ("rowbytes", {"rowbytes": (8 + W) * 4 - 4}),
        ("frame stride", {"stride": (6 + H) * 640 - 4}),
        ("RGBA origin", {"screen": base + 2}),
        ("NULL tables", {"tables": None}),
        ("tables not 16-byte aligned", {"tables": tab + 4}),
        ("table stride below 1024", {"table_stride": 1008}),
        ("table stride not a multiple of 16", {"table_stride": 1028}),
        ("table stride 4", {"table_stride": 4}),
    ]
    before = fe.launch_count
    for name, change in bad:
        assert call({**ok, **change}) == bb.E_INVALID, name
        assert fe.launch_count == before, name
    # Python: anything but a CUDA tensor of 4-byte elements shaped [256] or [N >= nframes, 256] is refused before the call
    t2 = torch.zeros((2, 256), dtype=torch.int32, device="cuda")
    wrong = [
        ("8-bit output", dict(rgba=False, tables=t2)),
        ("numpy", dict(rgba=True, tables=np.zeros((2, 256), np.uint32))),
        ("host tensor", dict(rgba=True, tables=t2.cpu())),
        ("2-byte elements", dict(rgba=True, tables=t2.to(torch.int16))),
        ("too few tables", dict(rgba=True, tables=t2[:1])),
        ("255 entries", dict(rgba=True, tables=t2[:, :255])),
        ("strided entries", dict(rgba=True, tables=torch.zeros((2, 512), dtype=torch.int32, device="cuda")[:, ::2])),
        ("3-D", dict(rgba=True, tables=t2[None])),
    ]
    for name, kw in wrong:
        with pytest.raises(ValueError):
            fe.warp_view(d_faces, base, x0=8, y0=6, rowbytes=640, nframes=2, screen_stride=120 * 640, **kw)
        assert fe.launch_count == before, name
    # the same arguments made valid do launch
    assert call(ok) == bb.OK
    assert call({**ok, "table_stride": 0}) == bb.OK
    fe.warp_view(d_faces, base, x0=8, y0=6, rowbytes=640, nframes=2, screen_stride=120 * 640, rgba=True, tables=t2,
                 stream=stream_of(torch))
    torch.cuda.synchronize()
    assert fe.launch_count > before
