"""What a lensmap install keeps and what it replaces, on the GPU.

The background stays, contents and all, across a rebuild at the same view size, and starts from zeros at a new view
size, also when a captured graph still reads the old one.  A graph keeps rendering the map, plan and background it
captured whichever way the old and the new map were made (host-planned or GPU-planned), until release_captures.
blinky_set_palette after a GPU-planned map changes the LUTs and nothing else.  Every warp is compared with the
oracle's render of the context's own map."""
import numpy as np
import pytest

from test_gpu_supplied_lensmap import built_map

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch(cuda_device):
    import torch

    return torch


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


def build(fe, lens, zoom, size, globe="cube"):
    fe.command(f"f_globe {globe}")
    fe.command(f"f_lens {lens}")
    fe.command(zoom)
    fe.build_lensmap(*size, 8)


def render(restate, fe, faces, palette, bg=None, rubix=False):
    """the oracle's render of the context's current map"""
    idx, tint = fe.lensmap()
    return restate.render(idx, tint, faces, restate.palmaps(palette), rubix, background=bg)


def unmapped(fe):
    return (fe.lensmap()[0] < 0).any()


def eager(torch, fe, d_faces):
    out = torch.full((fe.height, fe.width), 0x5A, dtype=torch.uint8, device="cuda")
    fe.warp(d_faces, out)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def capture(torch, fe, d_faces, out):
    fe.warp(d_faces, out)   # (eager first, as a host would)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fe.warp(d_faces, out)
    return g


def replay(torch, g, out):
    out.fill_(0x5A)
    g.replay()
    torch.cuda.synchronize()
    return out.cpu().numpy()


def cuda_map(torch, m):
    return torch.from_numpy(m.view(np.int32)).cuda()


def test_background_survives_a_same_size_rebuild(bb, fe, restate, palette, torch):
    size = (320, 200, 128)
    build(fe, "panini", "f_fov 180", size)
    bg = bb.synthetic_background(320, 200)
    fe.set_background(bg)
    build(fe, "fisheye1", "f_contain", size)
    assert unmapped(fe)
    faces = bb.synthetic_faces(fe.numplates, 128, 1)
    d_faces = torch.from_numpy(faces).cuda()
    assert np.array_equal(eager(torch, fe, d_faces), render(restate, fe, faces, palette, bg))


def test_a_view_change_zeroes_the_background(bb, fe, restate, palette, torch):
    # 320 x 200 and 250 x 256 have the same padded size: the background is zeroed in place
    build(fe, "fisheye1", "f_contain", (320, 200, 128))
    fe.set_background(bb.synthetic_background(320, 200))
    build(fe, "fisheye1", "f_contain", (250, 256, 128))
    assert unmapped(fe)
    faces = bb.synthetic_faces(fe.numplates, 128, 2)
    d_faces = torch.from_numpy(faces).cuda()
    assert np.array_equal(eager(torch, fe, d_faces), render(restate, fe, faces, palette))


def test_a_view_change_after_a_capture(bb, fe, restate, palette, torch):
    """the graph replays its own map and background, the eager warp starts from zeros and then from the background
    set after the rebuild, which the graph does not see"""
    build(fe, "fisheye1", "f_contain", (320, 200, 128))
    bg = bb.synthetic_background(320, 200)
    fe.set_background(bg)
    faces = bb.synthetic_faces(fe.numplates, 128, 3)
    d_faces = torch.from_numpy(faces).cuda()
    want_a = render(restate, fe, faces, palette, bg)
    out = torch.zeros((200, 320), dtype=torch.uint8, device="cuda")
    g = capture(torch, fe, d_faces, out)
    build(fe, "fisheye1", "f_contain", (250, 256, 128))
    assert unmapped(fe)
    assert np.array_equal(replay(torch, g, out), want_a)
    assert np.array_equal(eager(torch, fe, d_faces), render(restate, fe, faces, palette))
    bg_b = np.random.default_rng(9).integers(0, 256, (256, 250), dtype=np.uint8)
    fe.set_background(bg_b)
    assert np.array_equal(replay(torch, g, out), want_a)
    assert np.array_equal(eager(torch, fe, d_faces), render(restate, fe, faces, palette, bg_b))
    del g
    fe.release_captures()
    assert np.array_equal(eager(torch, fe, d_faces), render(restate, fe, faces, palette, bg_b))


def test_a_host_planned_capture_then_a_device_map(bb, fe, restate, palette, torch):
    W, H, ps = 160, 96, 64
    m1, n = built_map(bb, palette, "cube", "panini", "f_fov 180", (W, H, ps))
    m2, _ = built_map(bb, palette, "cube", "fisheye1", "f_contain", (W, H, ps))
    faces = bb.synthetic_faces(n, ps, 4)
    d_faces = torch.from_numpy(faces).cuda()
    fe.set_lensmap(m1, ps, n)
    want1 = render(restate, fe, faces, palette)
    out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    g = capture(torch, fe, d_faces, out)
    fe.set_lensmap(cuda_map(torch, m2), ps, n)
    want2 = render(restate, fe, faces, palette)
    assert not np.array_equal(want1, want2)
    assert np.array_equal(replay(torch, g, out), want1)
    assert np.array_equal(eager(torch, fe, d_faces), want2)
    del g
    fe.release_captures()
    assert np.array_equal(eager(torch, fe, d_faces), want2)


def test_a_device_planned_capture_then_a_build(bb, fe, restate, palette, torch):
    W, H, ps = 160, 96, 64
    m1, n = built_map(bb, palette, "cube", "panini", "f_fov 180", (W, H, ps))
    faces = bb.synthetic_faces(n, ps, 5)
    d_faces = torch.from_numpy(faces).cuda()
    fe.set_lensmap(cuda_map(torch, m1), ps, n)
    want1 = render(restate, fe, faces, palette)
    out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    g = capture(torch, fe, d_faces, out)
    build(fe, "fisheye1", "f_contain", (192, 120, ps))
    want2 = render(restate, fe, faces, palette)
    assert np.array_equal(replay(torch, g, out), want1)
    assert np.array_equal(eager(torch, fe, d_faces), want2)
    del g
    fe.release_captures()
    assert np.array_equal(eager(torch, fe, d_faces), want2)


def test_set_palette_after_a_device_map(bb, fe, restate, palette, torch):
    W, H, ps = 200, 120, 64
    m, n = built_map(bb, palette, "cube", "quincuncial", "f_cover", (W, H, ps), rubix=True)
    fe.set_rubix(True)
    fe.set_lensmap(cuda_map(torch, m), ps, n)
    assert (fe.lensmap()[1] != 255).any(), "the map has tinted pixels: the LUTs matter"
    faces = bb.synthetic_faces(n, ps, 6)
    d_faces = torch.from_numpy(faces).cuda()
    pal2 = bb.synthetic_palette(11)
    fe.set_palette(pal2)
    got = eager(torch, fe, d_faces)
    assert np.array_equal(got, render(restate, fe, faces, pal2, rubix=True))
    assert not np.array_equal(got, render(restate, fe, faces, palette, rubix=True))
    host = bb.Fisheye(device=None, palette=pal2)
    try:
        host.set_lensmap(m, ps, n)
        want, got = host.tile_plan(), fe.tile_plan()
        assert want[0].tobytes() == got[0].tobytes() and want[1].tobytes() == got[1].tobytes()
    finally:
        host.close()
