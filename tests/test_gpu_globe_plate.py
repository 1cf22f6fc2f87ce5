"""Device lensmap builds on globes that pick their plates with a `globe_plate` script (`fast`): every
translatable lens, the compiled reference's fixtures, custom globe_plate scripts, the module cache and one
full-size build, each against the interpreter build of the same context."""
import json
import os

import numpy as np
import pytest

from conftest import ALL_GLOBES, ALL_LENSES, sha
from test_globe_plate_transpile import CUSTOM_GLOBES, REFUSED_GLOBES, load_custom
from test_transpile import FORWARD_ONLY, TRANSLATABLE

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture()
def fe(bb, palette, cuda_device):
    f = bb.Fisheye(device=cuda_device, palette=palette)
    yield f
    f.close()


def build(fe, globe, lens, w, h, ps, threads):
    """the command sequence of test_host.py"""
    fe.clear_log()
    fe.command(f"f_globe {globe}")
    fe.command(f"f_lens {lens}")
    try:
        fe.build_lensmap(w, h, ps, threads)
        return 0
    except Exception as e:  # noqa: BLE001
        return e.code


@pytest.mark.gpu
@pytest.mark.parametrize("lens", TRANSLATABLE + FORWARD_ONLY)
def test_every_lens_on_fast_builds_on_the_device(fe, lens):
    forward = lens in FORWARD_ONLY
    for (w, h, ps), rubix in [((320, 200, 128), False), ((320, 200, 128), True), ((257, 131, 96), False), ((257, 131, 96), True)]:
        fe.command("f_globe fast")
        fe.command(f"f_lens {lens}")
        fe.set_rubix(rubix)
        fe.clear_log()
        fe.build_lensmap(w, h, ps, threads=0)
        info = fe.build_info
        assert info.startswith("device (forward):" if forward else "device:"), (lens, info)
        if forward:
            assert "texel owners" in info, info
        dev_idx, dev_tint = fe.lensmap()
        dev_disp, dev_log = fe.display(), fe.log
        fe.clear_log()
        fe.build_lensmap(w, h, ps, threads=1 if forward else -1)
        assert fe.build_info.startswith("host")
        idx, tint = fe.lensmap()
        assert np.array_equal(dev_idx, idx), (lens, w, rubix, int((dev_idx != idx).sum()), info)
        assert np.array_equal(dev_tint, tint), (lens, w, rubix, info)
        assert dev_disp == fe.display(), (lens, w, rubix)
        assert dev_log == fe.log, (lens, w, rubix)


@pytest.mark.gpu
def test_device_builds_reproduce_the_fast_golden_lensmaps(fe):
    lm = np.load(os.path.join(G, "lensmaps_small.npz"))
    meta = json.load(open(os.path.join(G, "meta_small.json")))
    W, H, PS = 128, 96, 48
    checked = 0
    for key in sorted(meta):  # every build, in test_host.py's order: later globes see earlier plate slots
        g, l = key.split("__")
        rc = build(fe, g, l, W, H, PS, 0 if g == "fast" else 1)
        if g != "fast":
            continue
        assert rc == 0 if meta[key]["rc"] == 0 else rc != 0, key
        assert fe.build_info.startswith("host" if l == "debug" else "device"), (key, fe.build_info)
        idx, tint = fe.lensmap()
        assert np.array_equal(idx, lm[key + "__idx"]), key
        assert np.array_equal(tint, lm[key + "__tint"]), key
        assert fe.scale == meta[key]["scale"] and fe.display() == meta[key]["display"], key
        assert sha(fe.plates()) == meta[key]["plates_sha"], key
        assert fe.log == meta[key]["log"], key
        checked += 1
    assert checked == 5


@pytest.mark.gpu
def test_device_builds_reproduce_the_fast_reference_digests(fe):
    want = json.load(open(os.path.join(G, "reference_digests.json")))["all_combinations_96x64x40"]
    W, H, PS = 96, 64, 40
    ways = {}
    for g in ALL_GLOBES:
        for l in ALL_LENSES:
            build(fe, g, l, W, H, PS, 0 if g == "fast" else 1)
            if g != "fast":
                continue
            r = want[f"{g}__{l}"]
            idx, tint = fe.lensmap()
            assert sha(idx, tint, fe.plates()) == r["maps"], (g, l, fe.build_info)
            assert r["display"] == fe.display() and r["scale"] == fe.scale, (g, l)
            assert r["log"] == fe.log, (g, l)
            way = fe.build_info.split(":")[0].split(" ")[0]
            ways[way] = ways.get(way, 0) + 1
    assert ways == {"device": len(ALL_LENSES) - 1, "host": 1}, ways  # debug is outside the subset


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CUSTOM_GLOBES))
def test_custom_globe_plate_device_build_equals_host(fe, name):
    """maps only: a map that points at plates >= numplates is not for warping (the faces hold numplates plates)"""
    for (w, h, ps), rubix in [((320, 200, 128), False), ((257, 131, 96), True)]:
        load_custom(fe, name)
        fe.set_rubix(rubix)
        fe.build_lensmap(w, h, ps, threads=0)
        info = fe.build_info
        assert info.startswith("device:"), (name, info)
        dev_idx, dev_tint = fe.lensmap()
        fe.build_lensmap(w, h, ps, threads=-1)
        idx, tint = fe.lensmap()
        assert np.array_equal(dev_idx, idx), (name, int((dev_idx != idx).sum()), info)
        assert np.array_equal(dev_tint, tint), (name, info)


@pytest.mark.gpu
@pytest.mark.parametrize("src, why", REFUSED_GLOBES)
def test_untranslatable_globe_plate_falls_back_with_its_reason(fe, src, why):
    fe.load_globe("t", src)
    fe.command("f_lens equirect")
    fe.build_lensmap(160, 100, 64, threads=0)
    assert fe.build_info.startswith("host (globe_plate: "), fe.build_info
    a = fe.lensmap_packed().copy()
    fe.build_lensmap(160, 100, 64, threads=-1)
    assert np.array_equal(a, fe.lensmap_packed())


@pytest.mark.gpu
def test_module_cache_sees_the_globe(bb, fe):
    w, h, ps = 320, 200, 128
    fe.command("f_globe fast")
    fe.command("f_lens panini")
    fe.build_lensmap(w, h, ps, threads=0)
    assert fe.build_info.startswith("device:")
    first = fe.lensmap_packed().copy()
    src = open(os.path.join(bb.SCRIPT_DIR, "lua-scripts", "globes", "fast.lua")).read()
    assert "local big_fov = 160" in src
    fe.load_globe("fast", src.replace("local big_fov = 160", "local big_fov = 120"))
    fe.build_lensmap(w, h, ps, threads=0)
    assert fe.build_info.startswith("device:"), fe.build_info
    dev = fe.lensmap_packed().copy()
    assert not np.array_equal(dev, first)
    fe.build_lensmap(w, h, ps, threads=-1)
    assert np.array_equal(dev, fe.lensmap_packed())


@pytest.mark.gpu
def test_full_size_fast_panini_equals_host(fe):
    fe.command("f_globe fast")
    fe.command("f_lens panini")
    fe.command("f_fov 180")
    fe.build_lensmap(3840, 2160, 2048, threads=0)
    assert fe.build_info.startswith("device:"), fe.build_info
    dev = fe.lensmap_packed().copy()
    fe.build_lensmap(3840, 2160, 2048, threads=-1)
    assert fe.build_info.startswith("host")
    assert np.array_equal(dev, fe.lensmap_packed())
