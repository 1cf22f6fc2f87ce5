"""Generates the committed golden vectors from the COMPILED REFERENCE (oracle/_ref,
i.e. the unmodified engine/NQ/fisheye.c of the original project) driving the repo's own
script set.  Needs oracle/_ref, built by build() with BLINKY_REFERENCE set:

    python tests/golden/make_golden.py

Outputs (all under tests/golden/):
  lensmaps_small.npz   idx/tint per (globe, lens) at 128x96, plates 48
  meta_small.json      scale, display flags, plate count, console log per combo
  c1.npz / c1.json     BASELINE config C1 (640x480, cube 6x256^2, panini f_fov 180):
                       lensmap + sha256 of rendered frames (rubix off / on)
  frames_small.npz     render_lensmap outputs for seeded faces/background, incl. a view
                       rectangle inside a wider screen (rowbytes > width)
  engine_frame.npz     whole F_RenderView frames (platesize = min(w,h))
  palmaps.npz          the six rubix LUTs for the seeded palette
  config.txt           F_WriteConfig output

The tests compare against these files; they do not need the reference.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import blinky_b200 as bb  # noqa: E402  (inputs only: seeded palette/faces/background, script dir)
from oracle.pyoracle import RefOracle  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

LENSES = ["cube", "cubestereo", "cylinder", "debug", "eckert1", "eckert4", "eckert5", "equirect", "fahey", "fisheye1",
          "fisheye2", "gallstereo", "gins8", "gumby", "hammer", "kavrayskiy7", "larrivee", "mercator", "miller",
          "mollweide", "panini", "polyconic", "quincuncial", "rectilinear", "sinusoidal", "stereographic",
          "vandergrinten", "wagner6", "winkel1", "winkel2", "winkeltripel"]
GLOBES = ["cube", "cube_corner", "cube_edge", "fast", "tetra", "trism"]
SMALL = (128, 96, 48)


def small_combos():
    combos = [("cube", l) for l in LENSES]
    for g in GLOBES[1:]:
        for l in ("panini", "quincuncial", "debug", "stereographic", "sinusoidal"):
            combos.append((g, l))
    return combos


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    pal = bb.synthetic_palette()
    R = RefOracle.get(bb.SCRIPT_DIR, pal)
    np.savez_compressed(os.path.join(OUT, "palmaps.npz"), palette=pal, palmaps=R.palmaps())

    # ---- small lensmaps ---------------------------------------------------
    W, H, PS = SMALL
    R.set_screen(W, H)
    arrays, meta = {}, {}
    for g, l in small_combos():
        R.clear_log()
        R.command(f"f_globe {g}")
        R.command(f"f_lens {l}")
        rc = R.build(W, H, PS)
        idx, tint = R.lensmap()
        key = f"{g}__{l}"
        arrays[key + "__idx"] = idx
        arrays[key + "__tint"] = tint
        meta[key] = dict(rc=rc, scale=R.scale, display=R.display(), numplates=R.numplates, map_type=R.map_type,
                         log=R.log, plates_sha=sha(R.plates()))
    np.savez_compressed(os.path.join(OUT, "lensmaps_small.npz"), **arrays)
    json.dump(meta, open(os.path.join(OUT, "meta_small.json"), "w"), indent=1, sort_keys=True)

    # ---- rendered frames (small) -------------------------------------------
    frames = {}
    for g, l, rubix in [("cube", "panini", False), ("cube", "panini", True), ("cube", "hammer", True),
                        ("trism", "stereographic", True), ("cube", "winkel1", True), ("fast", "quincuncial", False)]:
        R.command(f"f_globe {g}")
        R.command(f"f_lens {l}")
        if R.rubix_enabled != rubix:
            R.command("f_rubix")
        # view rectangle inside a wider screen: rowbytes 160, vrect at (8, 6)
        R.set_screen(160, 120, 160, 8, 6, W, H)
        R.build(W, H, PS)
        faces = bb.synthetic_faces(R.numplates, PS, 0)
        bg = np.random.default_rng(3).integers(0, 256, (120, 160), dtype=np.uint8)
        out = R.render(faces, bg)
        frames[f"{g}__{l}__rubix{int(rubix)}"] = out
    if R.rubix_enabled:
        R.command("f_rubix")
    np.savez_compressed(os.path.join(OUT, "frames_small.npz"), **frames)

    # ---- whole engine frames through F_RenderView ---------------------------
    eng = {}
    for g, l in [("cube", "panini"), ("cube", "fisheye1"), ("trism", "equirect")]:
        w, h = 96, 64
        R.set_screen(w, h)
        R.command(f"f_globe {g}")
        R.command(f"f_lens {l}")
        ps = min(w, h)
        faces = bb.synthetic_faces(R.numplates, ps, 1)
        bg = bb.synthetic_background(w, h)
        out, ncalls = R.frame(faces, bg)
        eng[f"{g}__{l}"] = out
        eng[f"{g}__{l}__calls"] = np.array([ncalls])
    np.savez_compressed(os.path.join(OUT, "engine_frame.npz"), **eng)

    # ---- C1 -----------------------------------------------------------------
    W1, H1, PS1 = 640, 480, 256
    R.set_screen(W1, H1)
    R.command("f_globe cube")
    R.command("f_lens panini")
    R.command("f_fov 180")
    R.command("f_rubixgrid 10 4 1")
    R.build(W1, H1, PS1)
    idx, tint = R.lensmap()
    faces = bb.synthetic_faces(6, PS1, 0)
    bg = bb.synthetic_background(W1, H1)
    off = R.render(faces, bg)
    R.command("f_rubix")
    on = R.render(faces, bg)
    R.command("f_rubix")
    np.savez_compressed(os.path.join(OUT, "c1.npz"), idx=idx, tint=tint)
    json.dump(dict(scale=R.scale, display=R.display(), idx_sha=sha(idx), tint_sha=sha(tint), faces_sha=sha(faces),
                   bg_sha=sha(bg), render_rubix_off_sha=sha(off), render_rubix_on_sha=sha(on),
                   mapped=int((idx >= 0).sum())),
              open(os.path.join(OUT, "c1.json"), "w"), indent=1, sort_keys=True)

    # ---- config ---------------------------------------------------------------
    R.command("f_lens hammer")
    R.command("f_globe trism")
    R.command("f_fov 123")
    R.command("f_rubixgrid 7 3.5 0.25")
    txt = R.write_config("/tmp/_blinky_cfg.txt")
    open(os.path.join(OUT, "config.txt"), "w").write(txt)
    R.command("f_rubixgrid 10 4 1")
    print("golden vectors written to", OUT)


if __name__ == "__main__":
    main()
