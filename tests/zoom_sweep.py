"""The zoom and view-shape sweep shared by the CPU and GPU sweep tests.

The zoom sets the lens's `scale`, and with it the range of every lens function: at the extremes `f_fov 360` sends panini
to infinity at the edge columns (scale comes out inf), `f_vfov 180` pushes mercator's sinh towards overflow, `f_fov`
near max_fov takes rectilinear and stereographic through tan near pi/2, and `f_cover` on a 1000 x 8 view stretches one
axis by two orders of magnitude.  These helpers list those cases once, lens-major, so that a lens's NVRTC units stay in
the device builder's cache for all of its zooms."""

# (width, height, platesize): odd (integer W/2), 16:9, very wide, very tall and tiny views, plate sizes 48 and 97
SHAPES = [(97, 61, 48), (97, 61, 97), (320, 180, 97), (1000, 8, 48), (8, 640, 97), (1, 1, 48), (3, 2, 97)]

# the reduced sweep for every globe but cube
REDUCED_GLOBES = ["cube_corner", "cube_edge", "tetra", "trism", "fast"]


def zoom_limits(fe, lens):
    """(max_fov, max_vfov) of `lens` as its script sets them (0 where it sets none); loads the lens"""
    fe.command(f"f_lens {lens}")
    return fe.max_fov, fe.max_vfov


def zooms(max_fov, max_vfov):
    """The zoom commands of the full sweep for a lens with these limits, without duplicates, in a fixed order.  The
    last ones, just past a limit, must be refused (so must every f_fov / f_vfov of a lens that sets no limits)."""
    out = []
    fovs = [1, 2, 45, 90, 179, 180, 181, max_fov - 1, max_fov]
    vfovs = [1, 90, max_vfov - 1, max_vfov]
    out += [f"f_fov {v}" for v in fovs if v > 0]
    out += [f"f_vfov {v}" for v in vfovs if v > 0]
    out += ["f_contain", "f_cover"]
    if max_fov > 0:
        out.append(f"f_fov {max_fov + 1}")
    if max_vfov > 0:
        out.append(f"f_vfov {max_vfov + 1}")
    seen = set()
    return [z for z in out if not (z in seen or seen.add(z))]


def reduced_cases(max_fov, max_vfov):
    """(zoom, (width, height, platesize)) of the reduced sweep: the zoom limits on a 97 x 61 view, f_cover on the very
    wide and very tall views"""
    out = []
    if max_fov > 0:
        out.append((f"f_fov {max_fov}", (97, 61, 48)))
    if max_vfov > 0:
        out.append((f"f_vfov {max_vfov}", (97, 61, 97)))
    out += [("f_cover", (1000, 8, 48)), ("f_cover", (8, 640, 97))]
    return out


def refused_past_the_limit(zoom, max_fov, max_vfov):
    """True for the zooms just past a limit, which every lens must refuse"""
    kind, _, value = zoom.partition(" ")
    return bool(value) and ((kind == "f_fov" and int(value) > max_fov) or (kind == "f_vfov" and int(value) > max_vfov))
