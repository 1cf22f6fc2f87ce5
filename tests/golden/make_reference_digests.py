"""Generates tests/golden/reference_digests.json: what the COMPILED REFERENCE (oracle/_ref) and the
reference's own Lua scripts produce in the comparisons of tests/test_host.py, tests/test_oracle.py and
tests/test_gpu_parity.py, so that those tests run without the reference.  Arrays are stored as
sha256 digests of their bytes (the tests compare them exactly), small values as they are.

    BLINKY_REFERENCE=<reference checkout> python -c "import __graft_entry__ as g; g.build()"
    python tests/golden/make_reference_digests.py <reference checkout>

The reference keeps its state in statics, and the tests drive it in one sequence; this script repeats
that sequence in one fresh process, in the order the suite runs it.
"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import blinky_b200 as bb  # noqa: E402
from conftest import ALL_GLOBES, ALL_LENSES, sha  # noqa: E402
from oracle.pyoracle import TRANSCRIBED_GLOBES, TRANSCRIBED_LENSES, RefOracle  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_digests.json")

CONSOLE_START = ("fisheye 1", "f_globe cube", "f_lens panini", "f_fov 180", "f_rubixgrid 10 4 1")
CONSOLE_SCRIPT = ["fisheye 1", "f_rubixgrid 10 4 1", "fisheye", "fisheye 0", "fisheye 1", "f_help", "f_rubix", "f_rubix", "f_rubixgrid",
                  "f_rubixgrid 7 3.5 0.25", "f_rubixgrid", "f_fov", "f_fov 100", "f_fov", "f_vfov 60", "f_vfov", "f_cover", "f_fov",
                  "f_contain", "f_fov", "f_lens", "f_globe", "f_lens hammer", "f_lens", "f_globe trism", "f_globe", "f_lens nosuchlens",
                  "f_globe nosuchglobe", "f_lens panini", "f_globe cube", "f_rubixgrid 10 4 1", "F_FOV 90"]
LIVE_COMBOS = [("cube", "panini", True), ("trism", "stereographic", False), ("tetra", "hammer", True),
               ("cube", "winkeltripel", True), ("fast", "panini", False), ("cube", "polyconic", True)]


def strip_errors(log):
    """file-open error lines: luaL_loadfile's text differs from the product's"""
    return "\n".join(x for x in log.split("\n") if not x.startswith("ERROR:"))


def build_host(fe, globe, lens, w, h, ps, threads):
    fe.clear_log()
    fe.command(f"f_globe {globe}")
    fe.command(f"f_lens {lens}")
    try:
        fe.build_lensmap(w, h, ps, threads)
        return 0
    except bb.BlinkyError as e:
        return e.code


def main(reference):
    pal = bb.synthetic_palette()
    R = RefOracle.get(bb.SCRIPT_DIR, pal)
    out = {}
    tmp = tempfile.mkdtemp()

    # test_host: every globe x lens
    W, H, PS = 96, 64, 40
    R.set_screen(W, H)
    combos = {}
    for g in ALL_GLOBES:
        for l in ALL_LENSES:
            R.clear_log()
            R.command(f"f_globe {g}")
            R.command(f"f_lens {l}")
            R.build(W, H, PS)
            idx, tint = R.lensmap()
            combos[f"{g}__{l}"] = dict(maps=sha(idx, tint, R.plates()), display=R.display(), scale=R.scale, log=R.log)
    out["all_combinations_96x64x40"] = combos

    # test_host: the product driven by the reference's script set
    own = {}
    with bb.Fisheye(device=None, basedir=os.path.join(reference, "game"), palette=pal) as a:
        for g in ALL_GLOBES:
            for l in ALL_LENSES:
                rc = build_host(a, g, l, 112, 80, 56, threads=4)
                idx, tint = a.lensmap()
                own[f"{g}__{l}"] = dict(rc=rc, maps=sha(idx, tint), scale=a.scale, display=a.display(), log=a.log,
                                        onload=a.onload, max_fov=a.max_fov, max_vfov=a.max_vfov, lens_width=a.lens_width,
                                        lens_height=a.lens_height, map_type=a.map_type)
    out["reference_scripts_112x80x56"] = own

    # test_host: console surface
    for c in CONSOLE_START:
        R.command(c)
    rubix = R.rubix_enabled
    R.clear_log()
    for c in CONSOLE_SCRIPT:
        R.command(c)
    out["console"] = dict(rubix_enabled=rubix, log=strip_errors(R.log), config=R.write_config(os.path.join(tmp, "cfg.txt")))

    # test_host: f_saveglobe PCX files
    w, h = 48, 40
    ps = min(w, h)
    R.set_screen(w, h)
    R.lib.ref_set_write_dir(tmp.encode())
    pcx = {}
    for globe in ("cube", "trism", "fast"):
        for margins in (0, 1):
            R.command(f"f_globe {globe}")
            R.command("f_lens equirect")
            faces = bb.synthetic_faces(R.numplates, ps, 6)
            R.command(f"f_saveglobe g{margins}_ {margins}")
            R.clear_log()
            R.frame(faces, bb.synthetic_background(w, h))
            files = []
            for i in range(R.numplates):
                files.append(sha(np.frombuffer(open(os.path.join(tmp, f"g{margins}_{i}.pcx"), "rb").read(), np.uint8)))
            pcx[f"{globe}__{margins}"] = dict(log=R.log, files=files)
    out["saveglobe_48x40"] = pcx

    # test_oracle: the restatement against the reference
    W, H, PS = 200, 150, 100
    R.set_screen(W, H)
    rest = {}
    for g in TRANSCRIBED_GLOBES:
        for l in TRANSCRIBED_LENSES:
            R.command(f"f_globe {g}")
            R.command(f"f_lens {l}")
            rc = R.build(W, H, PS)
            idx, tint = R.lensmap()
            rest[f"{g}__{l}"] = dict(rc=rc, scale=R.scale, maps=sha(idx, tint, R.plates()), display=R.display())
    out["restatement_200x150x100"] = rest

    # test_gpu_parity: rendered frames
    W, H, PS = 320, 200, 128
    R.set_screen(W, H)
    live = {}
    for g, l, rubix in LIVE_COMBOS:
        R.command(f"f_globe {g}")
        R.command(f"f_lens {l}")
        if R.rubix_enabled != rubix:
            R.command("f_rubix")
        R.build(W, H, PS)
        faces = bb.synthetic_faces(R.numplates, PS, 9)
        live[f"{g}__{l}__rubix{int(rubix)}"] = sha(R.render(faces, bb.synthetic_background(W, H)))
    if R.rubix_enabled:
        R.command("f_rubix")
    out["rendered_320x200x128"] = live

    json.dump(out, open(OUT, "w"), indent=0, sort_keys=True)
    print("reference digests written to", OUT)


if __name__ == "__main__":
    main(sys.argv[1])
