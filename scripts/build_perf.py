"""Lensmap build time: GPU (translated lens, NVRTC) vs interpreter on all usable CPUs.
Usage: python scripts/build_perf.py [W H PS] [LENS ...] [--globe NAME] [--host]
--globe picks the globe (default cube), e.g. fast, whose globe_plate script runs on the device too."""
import sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import blinky_b200 as bb

args = sys.argv[1:]
GLOBE = "cube"
if "--globe" in args:
    at = args.index("--globe")
    GLOBE = args[at + 1]
    del args[at:at + 2]
W, H, PS = (int(a) for a in args[0:3]) if len(args) >= 3 else (3840, 2160, 2048)
fe = bb.Fisheye(device=0, palette=bb.synthetic_palette())
print(f"usable cpus {bb.usable_cpus()}  size {W}x{H} ps {PS}")
LENSES = [a for a in args[3:] if not a.startswith("--")] or ["panini", "stereographic", "equirect", "hammer", "fisheye1", "mollweide", "vandergrinten", "winkeltripel", "eckert4", "quincuncial", "cube"]
for lens in LENSES:
    fe.command(f"f_globe {GLOBE}"); fe.command(f"f_lens {lens}")
    t = time.time(); fe.build_lensmap(W, H, PS, threads=0); t_first = time.time() - t
    info = fe.build_info
    a = fe.lensmap_packed().copy()
    fe.command(f"f_lens {lens}")
    t = time.time(); fe.build_lensmap(W, H, PS, threads=0); t_again = time.time() - t
    row = f"{lens:14s} gpu first {t_first*1e3:8.1f} ms  again {t_again*1e3:8.1f} ms  [{info}]"
    if "--host" in sys.argv:
        fe.command(f"f_lens {lens}")
        t = time.time(); fe.build_lensmap(W, H, PS, threads=-1); t_host = time.time() - t
        same = np.array_equal(a, fe.lensmap_packed())
        row += f"  host {t_host*1e3:8.1f} ms  identical={same}"
    print(row, flush=True)
