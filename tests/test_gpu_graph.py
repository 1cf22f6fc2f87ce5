"""The device warps captured into CUDA graphs (torch.cuda.graph, default capture mode), on the GPU.

Every replay is compared byte for byte with the eager warp of the same faces, which the rest of the suite pins to
the oracle and the golden frames; the dense 8-bit replays and the rebuild test are also compared with the CPU
oracle directly.  Before each replay the graph's static faces buffer gets new seeded frames, so a replay that
repeated the capture's work, skipped units or did some twice would show."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HAMMER = ("tetra", "hammer", "f_contain", (400, 226, 192), True)   # BOX, GATHER and EMPTY tiles, rubix overlay


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch

    return torch


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


def setup(fe, globe, lens, zoom, size, rubix):
    W, H, PS = size
    fe.command(f"f_globe {globe}")
    fe.command(f"f_lens {lens}")
    if zoom:
        fe.command(zoom)
    fe.set_rubix(rubix)
    fe.build_lensmap(W, H, PS, 8)


def faces_batch(bb, fe, n, seed):
    return np.stack([bb.synthetic_faces(fe.numplates, fe.platesize, seed + i) for i in range(n)])


def rgba_table():
    return np.random.default_rng(5).integers(0, 2**32, 256, dtype=np.uint64).astype(np.uint32)


class Target:
    """One warp call and the flat, random-filled device buffer it writes: dense frames ("dense"; "flat" through
    set_kernel(1)), or a view rectangle of screens ("view", "view-keep"; "odd-x0", which only the per-pixel kernel
    takes)."""

    KERNEL = {"dense": "warp_ring_kernel", "view": "warp_ring_kernel", "view-keep": "warp_ring_kernel",
              "flat": "warp_gather_kernel", "odd-x0": "warp_scalar_kernel"}

    def __init__(self, torch, fe, nframes, rgba, mode, seed, x0=None, screen_width=None):
        W, H = fe.width, fe.height
        self.bpp = 4 if rgba else 1
        self.fe, self.nframes, self.rgba, self.mode = fe, nframes, rgba, mode
        self.x0 = x0 if x0 is not None else (3 if mode == "odd-x0" else 8)
        self.y0 = 2
        sw = screen_width if screen_width is not None else 8 + W + 13
        self.rowbytes = -(-sw * self.bpp // 16) * 16
        self.fstride = W * H * self.bpp if mode in ("dense", "flat") else (self.y0 + H + 3) * self.rowbytes + 64
        gen = torch.Generator().manual_seed(seed)
        self.fill = torch.randint(0, 256, (nframes * self.fstride,), dtype=torch.uint8, generator=gen).cuda()
        self.buf = self.fill.clone()

    def warp(self, d_faces, buf=None, stream=None):
        buf = self.buf if buf is None else buf
        if self.mode in ("dense", "flat"):
            self.fe.set_kernel(1 if self.mode == "flat" else 0)
            self.fe.warp(d_faces, buf.data_ptr(), nframes=self.nframes, rgba=self.rgba, stream=stream)
            self.fe.set_kernel(0)
        else:
            self.fe.warp_view(d_faces, buf.data_ptr(), x0=self.x0, y0=self.y0, rowbytes=self.rowbytes, nframes=self.nframes,
                              keep_unmapped=self.mode == "view-keep", rgba=self.rgba, screen_stride=self.fstride,
                              stream=stream)

    def eager(self, torch, d_faces):
        out = self.fill.clone()
        self.warp(d_faces, out)
        torch.cuda.synchronize()
        return out


def capture(torch, fn, stream=None):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    return g


def oracle_frames(bb, restate, palette, fe, faces, rubix, bg):
    idx, tint = fe.lensmap()
    pm = restate.palmaps(palette)
    return np.stack([restate.render(idx, tint, faces[i], pm, rubix, background=bg) for i in range(len(faces))])


# ---- replay matches eager ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("rgba", [False, True])
@pytest.mark.parametrize("nframes", [1, 5, 16])
def test_replay_matches_eager(bb, fe, restate, palette, torch_mod, nframes, rgba):
    """1 and 5 frames: GATHER tiles as extra CTAs of the ring kernel's launch; 16 frames: the gather kernel in front
    and 16-frame units.  Dense, view and view with keep_unmapped on the ring kernel, the flat kernel, and a view
    at an odd x0 (per-pixel kernel); rubix on."""
    torch = torch_mod
    globe, lens, zoom, size, rubix = HAMMER
    setup(fe, globe, lens, zoom, size, rubix)
    bg = bb.synthetic_background(fe.width, fe.height)
    fe.set_background(bg)
    fe.set_rgba_table(rgba_table())
    d_faces = torch.from_numpy(faces_batch(bb, fe, nframes, 0)).cuda()
    seed = 100
    for mode in Target.KERNEL:
        tgt = Target(torch, fe, nframes, rgba, mode, seed=nframes + 7 * rgba)
        tgt.warp(d_faces)   # (eager first, as a host would)
        torch.cuda.synchronize()
        g = capture(torch, lambda: tgt.warp(d_faces))
        kernel = fe.last_kernel
        assert Target.KERNEL[mode] in kernel, (mode, kernel)
        if mode in ("dense", "view", "view-keep"):
            assert ("warp_tile_gather_kernel" in kernel) == (nframes > 8), kernel
        for _ in range(3):
            seed += 1
            faces = faces_batch(bb, fe, nframes, seed)
            d_faces.copy_(torch.from_numpy(faces))
            tgt.buf.copy_(tgt.fill)
            g.replay()
            want = tgt.eager(torch, d_faces)
            assert torch.equal(tgt.buf, want), (mode, nframes, rgba, seed, kernel)
            if mode == "dense" and not rgba:
                got = tgt.buf.cpu().numpy().reshape(nframes, fe.height, fe.width)
                assert np.array_equal(got, oracle_frames(bb, restate, palette, fe, faces, rubix, bg)), (nframes, seed)
        del g


# ---- schedules and streams ----------------------------------------------------------------------------------------

def test_all_ticket_schedule(bb, restate, palette, torch_mod, cuda_device, monkeypatch):
    """Every unit from the work counter, one frame per unit.  The capture stream has warped before; the graph is
    replayed five times, then eager warps run on the capture stream and on another stream: each launch must find
    its counter at zero."""
    torch = torch_mod
    monkeypatch.setenv("BLINKY_STATIC_PCT", "0")
    monkeypatch.setenv("BLINKY_FCHUNK", "1")
    globe, lens, zoom, size, rubix = HAMMER
    with bb.Fisheye(device=cuda_device, palette=palette) as f:   # the knobs are read when the context is created
        setup(f, globe, lens, zoom, size, rubix)
        bg = bb.synthetic_background(f.width, f.height)
        f.set_background(bg)
        N = 5
        d_faces = torch.from_numpy(faces_batch(bb, f, N, 0)).cuda()
        tgt = Target(torch, f, N, False, "dense", seed=1)
        cap, other = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        tgt.warp(d_faces, stream=cap.cuda_stream)
        torch.cuda.synchronize()
        g = capture(torch, lambda: tgt.warp(d_faces, stream=cap.cuda_stream), stream=cap)
        assert "warp_ring_kernel" in f.last_kernel, f.last_kernel
        for r in range(5):
            faces = faces_batch(bb, f, N, 200 + 10 * r)
            d_faces.copy_(torch.from_numpy(faces))
            tgt.buf.copy_(tgt.fill)
            g.replay()
            torch.cuda.synchronize()
            want = oracle_frames(bb, restate, palette, f, faces, rubix, bg)
            assert np.array_equal(tgt.buf.cpu().numpy().reshape(want.shape), want), ("replay", r)
            assert torch.equal(tgt.buf, tgt.eager(torch, d_faces)), ("replay vs eager", r)
        for s in (cap, other, cap):
            out = tgt.fill.clone()
            torch.cuda.synchronize()
            tgt.warp(d_faces, out, stream=s.cuda_stream)
            torch.cuda.synchronize()
            assert np.array_equal(out.cpu().numpy().reshape(want.shape), want), "eager after the replays"


def test_capture_on_a_fresh_stream(bb, fe, torch_mod):
    """A stream the context has never launched on: capturing there allocates nothing."""
    torch = torch_mod
    globe, lens, zoom, size, rubix = HAMMER
    setup(fe, globe, lens, zoom, size, rubix)
    d_faces = torch.from_numpy(faces_batch(bb, fe, 1, 0)).cuda()
    tgt = Target(torch, fe, 1, False, "dense", seed=2)
    tgt.warp(d_faces)
    torch.cuda.synchronize()
    fresh = torch.cuda.Stream()
    g = capture(torch, lambda: tgt.warp(d_faces, stream=fresh.cuda_stream), stream=fresh)
    for r in range(3):
        d_faces.copy_(torch.from_numpy(faces_batch(bb, fe, 1, 300 + r)))
        tgt.buf.copy_(tgt.fill)
        g.replay()
        assert torch.equal(tgt.buf, tgt.eager(torch, d_faces)), r


def test_two_graphs_replayed_concurrently(bb, fe, torch_mod):
    """Two graphs of one context, each warping into its own rectangle of one screen, replayed at the same time on
    two streams."""
    torch = torch_mod
    globe, lens, zoom, size, rubix = HAMMER
    setup(fe, globe, lens, zoom, size, rubix)
    W = fe.width
    left = Target(torch, fe, 1, False, "view-keep", seed=3, x0=4, screen_width=4 + 2 * W + 12)
    right = Target(torch, fe, 1, False, "view-keep", seed=3, x0=4 + W, screen_width=4 + 2 * W + 12)
    right.buf = left.buf   # one screen
    faces = [torch.from_numpy(faces_batch(bb, fe, 1, s)).cuda() for s in (0, 1)]
    for t, d in zip((left, right), faces):
        t.warp(d)
    torch.cuda.synchronize()
    graphs = [capture(torch, lambda t=t, d=d: t.warp(d)) for t, d in zip((left, right), faces)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for r in range(4):
        for i, d in enumerate(faces):
            d.copy_(torch.from_numpy(faces_batch(bb, fe, 1, 400 + 10 * r + i)))
        left.buf.copy_(left.fill)
        torch.cuda.synchronize()
        for g, s in zip(graphs, streams):
            with torch.cuda.stream(s):
                g.replay()
        torch.cuda.synchronize()
        want = left.fill.clone()
        left.warp(faces[0], want)
        right.warp(faces[1], want)
        torch.cuda.synchronize()
        assert torch.equal(left.buf, want), r


# ---- buffer lifetime ------------------------------------------------------------------------------------------------

def test_rebuild_after_capture(bb, fe, restate, palette, torch_mod):
    """Graphs captured with lens A (ring kernel and flat kernel) still render A after the context was rebuilt with
    lens B, at the same view size and then at another; eager warps render B; release_captures frees A's buffers."""
    assert hasattr(bb.Fisheye, "release_captures")   # without it a rebuild frees what the graphs read
    torch = torch_mod
    W, H, PS = 320, 200, 128
    setup(fe, "cube", "fisheye1", "f_contain", (W, H, PS), False)   # A: unmapped corners show the background
    bg = bb.synthetic_background(W, H)
    fe.set_background(bg)
    faces = faces_batch(bb, fe, 1, 0)
    d_faces = torch.from_numpy(faces).cuda()
    want_a = oracle_frames(bb, restate, palette, fe, faces, False, bg)
    targets = [Target(torch, fe, 1, False, mode, seed=4) for mode in ("dense", "flat")]
    graphs = []
    for t in targets:
        t.warp(d_faces)
        torch.cuda.synchronize()
        graphs.append(capture(torch, lambda t=t: t.warp(d_faces)))
    for size in ((W, H, PS), (256, 160, PS)):
        setup(fe, "cube", "panini", "f_fov 180", size, False)           # B
        bg_b = bg if size[0] == W else bb.synthetic_background(size[0], size[1])
        fe.set_background(bg_b)
        for t, g in zip(targets, graphs):
            t.buf.copy_(t.fill)
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(t.buf.cpu().numpy().reshape(want_a.shape), want_a), (t.mode, size)
        out = torch.zeros(size[0] * size[1], dtype=torch.uint8, device="cuda")
        fe.warp(d_faces, out)
        torch.cuda.synchronize()
        want_b = oracle_frames(bb, restate, palette, fe, faces, False, bg_b)
        assert np.array_equal(out.cpu().numpy().reshape(want_b.shape), want_b), size
    del graphs
    fe.release_captures()
    fe.warp(d_faces, out)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().reshape(want_b.shape), want_b)


# ---- the capture counter pool ---------------------------------------------------------------------------------------

POOL = 4096


def test_capture_pool_exhaustion_and_release(bb, fe, torch_mod):
    """Each captured ring kernel launch holds one of 4096 work counters until release_captures.  With none left a
    capture is refused with E_STATE and launches nothing; the flat kernel needs no counter; release_captures is
    refused while the capture is open, and afterwards gives all 4096 back."""
    torch = torch_mod
    setup(fe, "cube", "panini", None, (320, 200, 128), False)
    d_faces = torch.from_numpy(faces_batch(bb, fe, 1, 0)).cuda()
    tgt = Target(torch, fe, 1, False, "dense", seed=5)
    tgt.warp(d_faces)
    torch.cuda.synchronize()
    assert "warp_ring_kernel" in fe.last_kernel and "tile_gather" not in fe.last_kernel, fe.last_kernel
    want = tgt.eager(torch, d_faces)
    for attempt in range(2):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(POOL):
                tgt.warp(d_faces)
            before = fe.launch_count
            with pytest.raises(bb.BlinkyError) as e:
                tgt.warp(d_faces)
            assert e.value.code == bb.E_STATE and "blinky_release_captures" in str(e.value), str(e.value)
            assert fe.launch_count == before
            fe.set_kernel(1)
            fe.warp(d_faces, tgt.buf.data_ptr())
            fe.set_kernel(0)
            assert "warp_gather_kernel" in fe.last_kernel
            with pytest.raises(bb.BlinkyError) as e:
                fe.release_captures()
            assert e.value.code == bb.E_INVALID, (attempt, str(e.value))
        tgt.buf.copy_(tgt.fill)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(tgt.buf, want), attempt
        del g
        fe.release_captures()
