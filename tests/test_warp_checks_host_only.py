"""Which warp calls are accepted (check_warp, launch_plan.h, compiled here with g++) without a GPU: for every entry point
family — dense, view, view with tables, the ray warps at each filter and factor, blinky_ray_pyramid_bytes and
blinky_warp_host — every refusal's code and exact message, the precedence of each pair of adjacent checks, the values
derived for accepted calls, and the refusals of a NULL dense buffer and a negative blinky_warp_host origin."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_INVALID, E_CUDA, E_STATE = 0, -1, -5, -7
(INTERNAL, DENSE, DENSE_RGBA, VIEW, VIEW_RGBA, VIEW_TABLES, RAYS, RAYS_RGBA, RAYS_SS, RAYS_BILINEAR, RAYS_TRILINEAR, PYRAMID,
 HOST) = range(13)
NEAREST, BILINEAR, TRILINEAR = range(3)

# the call, the state and the derived values, as one flat int64 array each way
ARGS = ["entry", "faces", "face_stride", "out", "out_stride", "nframes", "rowbytes", "x0", "y0", "rgba", "tables", "table_stride",
        "dense_faces", "rays", "ray_stride", "xforms", "xform_stride", "factor", "filter", "scratch", "scratch_bytes",
        "W", "H", "ps", "globe_valid", "plate_script", "plates", "layout_rowbytes", "nlayout"]
OUTS = ["launch", "view", "pitch", "use_layout", "layout_rows", "lmax", "pyramid_bytes", "lay_rowbytes", "lay_ps"] + [f"base{i}" for i in range(6)]

SHIM = r"""
#include "launch_plan.h"
using namespace blinky;
extern "C" int check(const int64_t *a, const int *display, const int *rect, const int32_t *origins, char *why, size_t whylen, int64_t *o) {
    WarpRequest r(reinterpret_cast<const void *>(a[1]), a[2], reinterpret_cast<void *>(a[3]), a[4], static_cast<int>(a[5]), nullptr);
    r.entry = static_cast<WarpEntry>(a[0]);
    r.rowbytes = static_cast<int>(a[6]), r.x0 = static_cast<int>(a[7]), r.y0 = static_cast<int>(a[8]);
    r.rgba = a[9] != 0;
    r.tables = reinterpret_cast<const uint32_t *>(a[10]), r.table_stride = a[11];
    r.dense_faces = a[12] != 0;
    RayRequest q = {reinterpret_cast<const float *>(a[13]), static_cast<size_t>(a[14]), reinterpret_cast<const float *>(a[15]), static_cast<size_t>(a[16])};
    q.factor = static_cast<int>(a[17]), q.filter = static_cast<RayFilter>(a[18]);
    q.scratch = reinterpret_cast<void *>(a[19]), q.scratch_bytes = a[20];
    WarpState s;
    s.width = static_cast<int>(a[21]), s.height = static_cast<int>(a[22]), s.platesize = static_cast<int>(a[23]);
    s.display = display;
    s.plate_rect = reinterpret_cast<const int (*)[4]>(rect);
    s.globe.valid = a[24] != 0, s.globe.plate_script = a[25] != 0, s.globe.plates = static_cast<int>(a[26]);
    s.layout_rowbytes = static_cast<int>(a[27]), s.layout_origins = origins, s.layout_plates = static_cast<int>(a[28]);
    CheckedWarp c;
    std::string w;
    const int rc = check_warp(r, q, s, &c, &w);
    snprintf(why, whylen, "%s", w.c_str());
    const int64_t v[9] = {c.launch, reinterpret_cast<int64_t>(c.view), static_cast<int64_t>(c.pitch), c.use_layout, c.layout_rows, c.lmax,
                          static_cast<int64_t>(c.pyramid_bytes), c.layout.rowbytes, c.layout.ps};
    for (int i = 0; i < 9; ++i) o[i] = v[i];
    for (int i = 0; i < 6; ++i) o[9 + i] = static_cast<int64_t>(c.layout.plate_base[i]);
    return rc;
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("warp_checks")
    src = d / "shim.cpp"
    src.write_text(SHIM)
    so = d / "shim.so"
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-shared", "-fPIC", "-I", os.path.join(ROOT, "blinky_b200", "csrc"),
                        "-o", str(so), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:3000]
    so_lib = ctypes.CDLL(str(so))
    so_lib.check.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_size_t, ctypes.c_void_p]
    return so_lib


W, H, PS = 64, 48, 32
RB, X0, Y0 = 4 * W + 64, 8, 4          # an RGBA screen's rows, and the view's origin in it
STATE = dict(W=W, H=H, ps=PS, globe_valid=1, plate_script=0, plates=6, layout_rowbytes=0, nlayout=0, display=[1] * 6,
             rect=[[0, 0, PS - 1, PS - 1]] * 6, origins=[])
ATLAS = [(c * PS, r * PS) for r in range(2) for c in range(3)]
FAMILY = {
    "dense": dict(entry=DENSE, out_stride=W * H),
    "dense_rgba": dict(entry=DENSE_RGBA, rgba=1, out_stride=4 * W * H),
    "internal": dict(entry=INTERNAL, out_stride=W * H, dense_faces=1),
    "view": dict(entry=VIEW, rowbytes=W + 16, x0=X0, y0=Y0, out_stride=(W + 16) * (H + Y0)),
    "view_rgba": dict(entry=VIEW_RGBA, rgba=1, rowbytes=RB, x0=X0, y0=Y0, out_stride=RB * (H + Y0)),
    "view_tables": dict(entry=VIEW_TABLES, rgba=1, rowbytes=RB, x0=X0, y0=Y0, out_stride=RB * (H + Y0), tables=0x30000, table_stride=1024),
    "rays": dict(entry=RAYS, rowbytes=W + 16, x0=X0, y0=Y0, out_stride=(W + 16) * (H + Y0), rays=0x40000, xforms=0x50000),
    "rays_rgba": dict(entry=RAYS_RGBA, rgba=1, rowbytes=RB, x0=X0, y0=Y0, out_stride=RB * (H + Y0), rays=0x40000, xforms=0x50000),
    "rays_ss": dict(entry=RAYS_SS, rgba=1, rowbytes=RB, x0=X0, y0=Y0, out_stride=RB * (H + Y0), rays=0x40000, xforms=0x50000, factor=2),
    "rays_bilinear": dict(entry=RAYS_BILINEAR, rgba=1, rowbytes=RB, x0=X0, y0=Y0, out_stride=RB * (H + Y0), rays=0x40000, xforms=0x50000,
                          filter=BILINEAR),
    "rays_trilinear": dict(entry=RAYS_TRILINEAR, rgba=1, rowbytes=RB, x0=X0, y0=Y0, out_stride=RB * (H + Y0), rays=0x40000, xforms=0x50000,
                           filter=TRILINEAR, scratch=0x60000, scratch_bytes=1 << 20),
    "pyramid": dict(entry=PYRAMID),
    "host": dict(entry=HOST, rowbytes=W + 16, x0=X0, y0=Y0, out_stride=(W + 16) * (H + Y0)),
}
CALL = dict(faces=0x10000, face_stride=6 * PS * PS, out=0x20000, out_stride=0, nframes=2, rowbytes=0, x0=0, y0=0, rgba=0, tables=0, table_stride=0,
            dense_faces=0, rays=0, ray_stride=0, xforms=0, xform_stride=0, factor=1, filter=NEAREST, scratch=0, scratch_bytes=0)


def check(lib, family, **kw):
    a = dict(CALL, **STATE)
    a.update(FAMILY[family])
    a.update(kw)
    if a["origins"]:
        a["layout_rowbytes"] = a.get("layout_rowbytes") or 3 * PS
        a["nlayout"] = len(a["origins"])
    arr = (ctypes.c_int64 * len(ARGS))(*[a[k] for k in ARGS])
    display = (ctypes.c_int * 6)(*a["display"])
    rect = (ctypes.c_int * 24)(*[v for r in a["rect"] for v in r])
    origins = (ctypes.c_int32 * 12)(*[v for xy in a["origins"] for v in xy])
    why = ctypes.create_string_buffer(1024)
    out = (ctypes.c_int64 * len(OUTS))()
    rc = lib.check(arr, display, rect, origins, why, 1024, out)
    return rc, why.value.decode(), dict(zip(OUTS, out))


def refusal(lib, family, **kw):
    rc, why, _ = check(lib, family, **kw)
    return rc, why


VIEWS = ["view", "view_rgba", "view_tables", "rays", "rays_rgba", "rays_ss", "rays_bilinear", "rays_trilinear"]
RAYS_ALL = ["rays", "rays_rgba", "rays_ss", "rays_bilinear", "rays_trilinear"]
NAME = {"dense": "blinky_warp_device", "dense_rgba": "blinky_warp_device_rgba", "internal": "warp", "view": "blinky_warp_device_view",
        "view_rgba": "blinky_warp_device_view_rgba", "view_tables": "blinky_warp_device_view_rgba_tables", "rays": "blinky_warp_device_rays",
        "rays_rgba": "blinky_warp_device_rays_rgba", "rays_ss": "blinky_warp_device_rays_supersampled",
        "rays_bilinear": "blinky_warp_device_rays_bilinear", "rays_trilinear": "blinky_warp_device_rays_trilinear",
        "pyramid": "blinky_ray_pyramid_bytes"}
NO_LENSMAP = dict(W=0, H=0, ps=0)
PYRAMID_32 = (4 * 6 * (16 * 16 + 8 * 8 + 4 * 4 + 2 * 2 + 1) + 255) // 256 * 256   # levels 1..5 of 6 plates of 32 texels


def test_every_family_accepts_its_base_call(lib):
    for family in FAMILY:
        rc, why, out = check(lib, family)
        assert (rc, why) == (OK, ""), family
        assert out["launch"] == (family != "pyramid"), family


# ---- refusals: code and message, per family ---------------------------------------------------------------------------

def cases():
    """(family, call, code, message) of every refusal"""
    out = []
    layout_msgs = [
        (dict(origins=ATLAS[:5] + [(2 * PS + 8, PS)]), E_INVALID, f"face layout: plate 5 at x = {2 * PS + 8} does not fit rowbytes {3 * PS} with plate size {PS}"),
        (dict(origins=ATLAS[:4], display=[1, 1, 1, 1, 0, 0], rect=[[0, 0, PS - 1, PS - 1]] * 4 + [[1, 1, 0, 0]] * 2, face_stride=6 * PS * PS - 1),
         E_INVALID, f"face layout: face_stride {6 * PS * PS - 1} is smaller than a frame's surface ({2 * PS} rows of {3 * PS} bytes)"),
    ]
    for f in ["dense", "dense_rgba", "view", "view_rgba", "view_tables", "host"]:
        out.append((f, dict(origins=ATLAS[:4]), E_INVALID, "face layout: the lensmap samples plate 4, which has no origin (the layout has 4)"))
        out += [(f, kw, code, msg) for kw, code, msg in layout_msgs]
    for f in RAYS_ALL:
        out.append((f, dict(origins=ATLAS[:4], display=[1, 1, 1, 1, 0, 0], rect=[[0, 0, PS - 1, PS - 1]] * 4 + [[1, 1, 0, 0]] * 2), E_INVALID,
                    "face layout: the globe has plate 4, which has no origin (the layout has 4)"))
        out += [(f, dict(kw, plates=4), code, msg) for kw, code, msg in layout_msgs]
    for f in VIEWS:
        n = NAME[f]
        rb = FAMILY[f]["rowbytes"]
        out += [
            (f, dict(faces=0), E_INVALID, f"{n}: NULL buffer"),
            (f, dict(out=0), E_INVALID, f"{n}: NULL buffer"),
            (f, dict(x0=-1), E_INVALID, f"{n}: the view origin (x0, y0) must not be negative"),
            (f, dict(y0=-1), E_INVALID, f"{n}: the view origin (x0, y0) must not be negative"),
            (f, dict(rowbytes=(X0 + W) * (4 if FAMILY[f].get("rgba") else 1) - 1), E_INVALID, f"{n}: rowbytes too small for the view rectangle"),
            (f, dict(out_stride=(H + Y0) * rb - 1), E_INVALID, f"{n}: screen_frame_stride too small for the view rectangle"),
            (f, dict(rowbytes=1 << 27, out_stride=(H + Y0) << 27), E_INVALID, "warp: the output row pitch must hold a row of the view and be at most 64 MB"),
        ]
        if FAMILY[f].get("rgba"):
            msg = f"{n}: the RGBA view origin, rowbytes and screen_frame_stride must be 4-byte aligned"
            out += [(f, dict(out=0x20002), E_INVALID, msg), (f, dict(rowbytes=RB + 2, out_stride=(RB + 2) * (H + Y0)), E_INVALID, msg),
                    (f, dict(out_stride=RB * (H + Y0) + 2), E_INVALID, msg)]
        if f == "view_tables" or f in RAYS_ALL[1:]:
            out += [(f, dict(tables=0x30008), E_INVALID, f"{n}: d_tables must be a non-NULL, 16-byte aligned device pointer")]
            msg = f"{n}: table_stride must be 0 (one table for every frame) or at least 1024, a multiple of 16 and below 16 GB"
            out += [(f, dict(tables=0x30000, table_stride=s), E_INVALID, msg) for s in (1008, 1032, 16 << 32)]
        if f == "view_tables":
            out.append((f, dict(tables=0), E_INVALID, f"{n}: d_tables must be a non-NULL, 16-byte aligned device pointer"))
        if f in VIEWS[:3]:
            out += [(f, dict(nframes=65536), E_INVALID, "warp: at most 65535 frames per launch"),
                    (f, NO_LENSMAP, E_CUDA, "warp: no lensmap on the device (call blinky_build_lensmap)")]
    for f in RAYS_ALL:
        n = NAME[f]
        factor = FAMILY[f].get("factor", 1)
        out += [
            (f, NO_LENSMAP, E_STATE, f"{n}: no lensmap installed (the view's size and background are the installed lensmap's)"),
            (f, dict(globe_valid=0), E_STATE, f"{n}: no valid globe"),
            (f, dict(plate_script=1), E_STATE, f"{n}: the globe picks its plates with a globe_plate script, whose decisions can need the interpreter: "
                                              "map such rays with blinky_set_raymap_device and warp the installed lensmap"),
            (f, dict(rays=0), E_INVALID, f"{n}: NULL rays"),
            (f, dict(rays=0x40002), E_INVALID, f"{n}: d_rays and d_xforms must be 4-byte aligned"),
            (f, dict(xforms=0x50002), E_INVALID, f"{n}: d_rays and d_xforms must be 4-byte aligned"),
            (f, dict(xform_stride=32), E_INVALID, f"{n}: xform_stride must be 0 (one matrix for every frame) or a multiple of 4 of at least 36"),
            (f, dict(xform_stride=38), E_INVALID, f"{n}: xform_stride must be 0 (one matrix for every frame) or a multiple of 4 of at least 36"),
            (f, dict(nframes=65536), E_INVALID, f"{n}: at most 65535 frames per launch"),
            (f, dict(W=W, H=H, ps=6689), E_STATE, "warp_rays: the installed lensmap's plate size 6689 is beyond what a ray map takes "
                                                  "(6 * platesize^2 must fit the 28-bit texel index)"),
        ]
        field = "factor^2 * width * height" if f in ("rays_ss", "rays_bilinear") else "width * height"
        msg = f"{n}: ray_stride must be 0 (one field for every frame) or a multiple of 4 of at least 12 * {field}"
        out += [(f, dict(ray_stride=12 * factor * factor * W * H - 4), E_INVALID, msg), (f, dict(ray_stride=12 * factor * factor * W * H + 2), E_INVALID, msg)]
        if f != "rays" and f != "rays_rgba":
            big = dict(W=46341, H=46341, rowbytes=4 * (X0 + 46341), out_stride=4 * (X0 + 46341) * (Y0 + 46341))
            out.append((f, big, E_INVALID, "warp_rays: a field of factor^2 * width * height = "
                                           f"{factor * factor * 46341 * 46341} pixels is beyond the kernel's 31-bit pixel index"))
    for k in (0, 5):
        out.append(("rays_bilinear", dict(factor=k), E_INVALID, "blinky_warp_device_rays_bilinear: factor must be 1, 2, 3 or 4"))
    for k in (1, 5):
        out.append(("rays_ss", dict(factor=k), E_INVALID, "blinky_warp_device_rays_supersampled: factor must be 2, 3 or 4"))
    tri = "rays_trilinear"
    out += [(tri, dict(scratch=0), E_INVALID, f"warp_rays: NULL scratch (the frames' pyramids need {PYRAMID_32} bytes each)"),
            (tri, dict(scratch=0x60008), E_INVALID, "warp_rays: the scratch must be 16-byte aligned"),
            (tri, dict(scratch_bytes=2 * PYRAMID_32 - 1), E_INVALID,
             f"warp_rays: scratch_bytes {2 * PYRAMID_32 - 1} is below nframes * {PYRAMID_32} (blinky_ray_pyramid_bytes)")]
    for f in ["dense", "dense_rgba", "internal"]:
        out += [(f, NO_LENSMAP, E_CUDA, "warp: no lensmap on the device (call blinky_build_lensmap)"),
                (f, dict(nframes=65536), E_INVALID, "warp: at most 65535 frames per launch"),
                (f, dict(faces=0), E_INVALID, f"{NAME[f]}: NULL buffer"),
                (f, dict(out=0), E_INVALID, f"{NAME[f]}: NULL buffer"),
                (f, dict(W=(1 << 26) + 4, H=1), E_INVALID, "warp: the output row pitch must hold a row of the view and be at most 64 MB")]
    msg = "blinky_warp_device_rgba: the RGBA view origin, rowbytes and screen_frame_stride must be 4-byte aligned"
    out += [("dense_rgba", dict(out=0x20002), E_INVALID, msg), ("dense_rgba", dict(out_stride=4 * W * H + 2), E_INVALID, msg)]
    out += [("pyramid", NO_LENSMAP, E_STATE, "blinky_ray_pyramid_bytes: no lensmap installed (its plate size sizes the pyramid)"),
            ("pyramid", dict(globe_valid=0), E_STATE, "blinky_ray_pyramid_bytes: no valid globe"),
            ("pyramid", dict(ps=6689), E_STATE, "blinky_ray_pyramid_bytes: the installed lensmap's plate size 6689 is beyond what the ray warps take "
                                                "(6 * platesize^2 must fit the 28-bit texel index)")]
    out += [("host", dict(faces=0), E_INVALID, "NULL buffer"), ("host", dict(out=0), E_INVALID, "NULL buffer"),
            ("host", dict(rowbytes=X0 + W - 1), E_INVALID, "dst_rowbytes too small for the view rectangle"),
            ("host", NO_LENSMAP, E_CUDA, "warp_host: no lensmap on the device (call blinky_build_lensmap)")]
    return out


CASES = cases()


@pytest.mark.parametrize("family,kw,code,msg", CASES, ids=[f"{c[0]}-{i}" for i, c in enumerate(CASES)])
def test_refusal(lib, family, kw, code, msg):
    assert refusal(lib, family, **kw) == (code, msg)


def test_every_family_has_refusals():
    assert {c[0] for c in CASES} == set(FAMILY)


# ---- precedence: a call failing two adjacent checks gets the earlier one ----------------------------------------------

def precedence():
    """(family, [call failing check i, ...]) in each family's order; each adjacent pair is tested together"""
    rb = dict(rowbytes=1)
    out = []
    for f in ["view", "view_rgba", "view_tables"]:
        steps = [dict(faces=0), dict(x0=-1), rb, dict(out_stride=1)]
        if f != "view":
            steps.append(dict(out=0x20002))
        if f == "view_tables":
            steps += [dict(tables=0x30008), dict(table_stride=8)]
        steps += [NO_LENSMAP, dict(nframes=65536), dict(rowbytes=1 << 27, out_stride=(H + Y0) << 27), dict(origins=ATLAS[:4])]
        out.append((f, steps))
    for f in RAYS_ALL:
        steps = [NO_LENSMAP, dict(globe_valid=0), dict(plate_script=1), dict(rays=0), dict(xforms=0x50002)]
        if f in ("rays_ss", "rays_bilinear"):
            steps.append(dict(factor=5))
        steps += [dict(ray_stride=4), dict(xform_stride=4), dict(nframes=65536), dict(faces=0), dict(x0=-1), rb, dict(out_stride=1)]
        if f != "rays":
            steps += [dict(out=0x20002), dict(tables=0x30008), dict(tables=0x30000, table_stride=8)]
        steps.append(dict(ps=6689))
        if f != "rays" and f != "rays_rgba":
            steps.append(dict(W=46341, H=46341, rowbytes=4 * (X0 + 46341), out_stride=4 * (X0 + 46341) * (Y0 + 46341)))
        if f == "rays_trilinear":
            steps += [dict(scratch=0), dict(scratch=0x60008), dict(scratch_bytes=1)]
        steps += [dict(rowbytes=1 << 27, out_stride=(H + Y0) << 27), dict(origins=ATLAS[:4])]
        out.append((f, steps))
    for f in ["dense", "dense_rgba", "internal"]:
        steps = [NO_LENSMAP, dict(nframes=65536), dict(out=0)]
        if f == "dense_rgba":
            steps.append(dict(out_stride=4 * W * H + 2))
        steps.append(dict(origins=ATLAS[:4]) if f != "internal" else dict(W=(1 << 26) + 4, H=1))
        out.append((f, steps))
    out.append(("pyramid", [NO_LENSMAP, dict(globe_valid=0), dict(ps=6689)]))
    out.append(("host", [dict(faces=0), dict(x0=-1), dict(rowbytes=1), NO_LENSMAP, dict(origins=ATLAS[:4])]))
    return out


def merge(a, b):
    """b's failure layered under a's, so that the call fails both"""
    m = dict(b)
    m.update(a)
    if "x0" in a and "rowbytes" in b:
        m["rowbytes"] = 1   # (x0 = -1 alone would make rowbytes 1 too small only for W > 2)
    if "W" in a and a["W"] == 0:   # no lensmap: the later checks of the view size see 0
        m.update(W=0, H=0, ps=0)
    return m


@pytest.mark.parametrize("family,steps", precedence(), ids=[p[0] for p in precedence()])
def test_precedence(lib, family, steps):
    for i in range(len(steps) - 1):
        first, second = steps[i], steps[i + 1]
        alone = refusal(lib, family, **first)
        assert alone[0] != OK, (family, first)
        assert refusal(lib, family, **second)[0] != OK, (family, second)
        both = refusal(lib, family, **merge(first, second))
        assert both == alone, (family, first, second)


def test_zero_frames_launch_nothing_after_the_checks_before_them(lib):
    for f in FAMILY:
        if f == "pyramid":
            continue
        rc, why, out = check(lib, f, nframes=0)
        assert (rc, why, out["launch"]) == (OK, "", 0), f
    # ... but only after them: the view checks come first, the dense ones' after; blinky_warp_host checks its layout
    assert refusal(lib, "view", nframes=0, x0=-1)[0] == E_INVALID
    assert refusal(lib, "dense", nframes=0, out=0) == (OK, "")
    assert refusal(lib, "rays", nframes=0, ps=6689) == (OK, "")
    assert refusal(lib, "host", nframes=0, origins=ATLAS[:4])[0] == E_INVALID


# ---- derived values ---------------------------------------------------------------------------------------------------

def test_view_origin_and_pitch(lib):
    for f in FAMILY:
        if f == "pyramid":
            continue
        rc, _, out = check(lib, f)
        assert rc == OK
        a = dict(CALL, **FAMILY[f])
        bpp = 4 if a["rgba"] else 1
        pitch = a["rowbytes"] if a["entry"] in (VIEW, VIEW_RGBA, VIEW_TABLES, RAYS, RAYS_RGBA, RAYS_SS, RAYS_BILINEAR, RAYS_TRILINEAR, HOST) else W * bpp
        assert out["pitch"] == pitch, f
        assert out["view"] == a["out"] + a["y0"] * pitch + a["x0"] * bpp, f


def test_face_layout(lib):
    for f in ["dense", "view_rgba", "host", "rays_rgba"]:
        rc, _, out = check(lib, f, origins=ATLAS, layout_rowbytes=3 * PS + 16, face_stride=2 * PS * (3 * PS + 16))
        assert rc == OK, f
        assert out["use_layout"] == 1 and out["layout_rows"] == 2 * PS and out["lay_rowbytes"] == 3 * PS + 16 and out["lay_ps"] == PS, f
        assert [out[f"base{i}"] for i in range(6)] == [y * (3 * PS + 16) + x for x, y in ATLAS], f
    # dense faces: none for the faces' warps (and warp_host's frames), the layout with rowbytes = ps for the ray warps
    _, _, out = check(lib, "internal", origins=ATLAS)
    assert out["use_layout"] == 0 and out["lay_rowbytes"] == 0
    _, _, out = check(lib, "view")
    assert out["use_layout"] == 0 and out["lay_rowbytes"] == 0
    _, _, out = check(lib, "rays")
    assert out["use_layout"] == 1 and out["lay_rowbytes"] == PS and out["layout_rows"] == 0
    assert [out[f"base{i}"] for i in range(6)] == [i * PS * PS for i in range(6)]
    # the plates a warp needs origins for: those the lensmap samples, or every plate of the globe for a ray warp
    sparse = dict(origins=ATLAS[:4], display=[1, 1, 1, 1, 0, 0], rect=[[0, 0, PS - 1, PS - 1]] * 4 + [[1, 1, 0, 0]] * 2)
    assert check(lib, "view", **sparse)[0] == OK
    assert check(lib, "rays", plates=4, **sparse)[0] == OK
    assert check(lib, "rays", **sparse)[0] == E_INVALID


def test_pyramid_levels(lib):
    _, _, out = check(lib, "rays_trilinear")
    assert (out["lmax"], out["pyramid_bytes"]) == (5, PYRAMID_32)
    _, _, out = check(lib, "pyramid", plates=4)
    assert (out["lmax"], out["pyramid_bytes"]) == (5, (4 * 4 * (256 + 64 + 16 + 4 + 1) + 255) // 256 * 256)
    # the other ray warps launch no pyramid
    for f in ["rays", "rays_rgba", "rays_ss", "rays_bilinear"]:
        assert check(lib, f)[2]["lmax"] == 0, f
    # the largest plate size a ray map takes
    assert check(lib, "pyramid", ps=6688)[0] == OK
    assert check(lib, "rays_trilinear", ps=6688, scratch_bytes=1 << 40)[0] == OK


# ---- the two refusals the parent lacked -------------------------------------------------------------------------------

def test_dense_null_buffers_are_refused(lib):
    for f in ["dense", "dense_rgba"]:
        for kw in (dict(faces=0), dict(out=0)):
            assert refusal(lib, f, **kw) == (E_INVALID, f"{NAME[f]}: NULL buffer")


def test_host_negative_origin_is_refused(lib):
    for kw in (dict(x0=-1), dict(y0=-1), dict(x0=-1, rowbytes=W - 1)):
        assert refusal(lib, "host", **kw) == (E_INVALID, "the view origin (x0, y0) must not be negative")
