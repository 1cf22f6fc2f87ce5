"""The device warps' launch decisions (launch_plan.h, compiled here with g++) without a GPU: the ticket schedule against
a simulation of the ring kernel's draw protocol, the kernel choice, frames per unit, the ring geometry, the gather
placement and the kernel variant's index and tags."""
import ctypes
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RING, VECTOR, SCALAR = 0, 1, 2   # WarpKernel: warp_ring_kernel, K1, K0

SHIM = r"""
#include "launch_plan.h"
using namespace blinky;
extern "C" int choose(int force_flat, int have_plan, int has_box, int w, int h, size_t opx, uintptr_t out, size_t pitch, size_t out_stride,
                      uintptr_t faces, size_t face_stride, int nframes, uint32_t rowbytes, const int32_t *origins, int nplates) {
    FaceLayoutParams lay = {};   // (choose_kernel reads rowbytes and the x origins)
    lay.rowbytes = rowbytes;
    for (int i = 0; i < nplates; ++i) lay.org_x[i] = origins[2 * i], lay.org_y[i] = origins[2 * i + 1];
    WarpRequest r(reinterpret_cast<const void *>(faces), face_stride, reinterpret_cast<void *>(out), out_stride, nframes, nullptr);
    r.rgba = opx == 4;
    return static_cast<int>(choose_kernel(r, pitch, rowbytes ? &lay : nullptr, w, h, have_plan != 0, has_box != 0, force_flat != 0));
}
extern "C" void geometry(size_t smem, int want, int merged, size_t fixed, uint32_t max_box, int override_bytes, int *warps, uint32_t *bytes) {
    const RingGeometry g = ring_geometry(smem, want, merged != 0, fixed, max_box, override_bytes);
    *warps = g.warps;
    *bytes = g.ring_bytes;
}
extern "C" int rides(uint32_t ngather, int nframes, int merged_items_max, int serial) {
    return gather_rides_along(ngather, nframes, merged_items_max, serial != 0);
}
extern "C" uint32_t items(uint32_t ngather, int nframes) { return gather_items(ngather, nframes); }
extern "C" uint32_t fpu(uint32_t ring_tiles, uint32_t nframes, uint32_t grid, int override_chunk) {
    return frames_per_unit(ring_tiles, nframes, grid, override_chunk);
}
extern "C" void tickets(uint32_t nunits, uint32_t grid, int pct, uint32_t *nstatic, uint32_t *ndraws) {
    const TicketSchedule s = ticket_schedule(nunits, grid, pct);
    *nstatic = s.nstatic;
    *ndraws = s.ndraws;
}
extern "C" int variant_index(int i) {
    const KernelVariant v = {(i & 1) != 0, (i & 2) != 0, (i & 4) != 0, (i & 8) != 0, (i & 16) != 0};
    return v.index();
}
extern "C" const char *variant_tags(int i) {
    const KernelVariant v = {(i & 1) != 0, (i & 2) != 0, (i & 4) != 0, (i & 8) != 0, (i & 16) != 0};
    return v.tags();
}
extern "C" int variant_exists(int i) { return KernelVariant::exists(i); }
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("launch_plan")
    src = d / "shim.cpp"
    src.write_text(SHIM)
    so = d / "shim.so"
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-shared", "-fPIC", "-I", os.path.join(ROOT, "blinky_b200", "csrc"),
                        "-o", str(so), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    so_lib = ctypes.CDLL(str(so))
    so_lib.choose.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t,
                              ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int]
    so_lib.geometry.argtypes = [ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_int,
                                ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint32)]
    so_lib.fpu.restype = ctypes.c_uint32
    so_lib.items.restype = ctypes.c_uint32
    so_lib.variant_tags.restype = ctypes.c_char_p
    return so_lib


# ---- ticket schedule -------------------------------------------------------------------------------------------------

def simulate(nunits, grid, nstatic, ndraws, rng):
    """warp_ring_kernel's work distribution with the warps' draws interleaved at random: warp w's k-th ticket is
    w + k*grid while k < nstatic; after that each ticket is one draw on the counter, made only while the warp's last
    ticket was good, and the draw that receives ndraws - 1 sets the counter back to 0 (ticket_drawn).  Returns the
    number of draws, how often each unit was taken and the counter at the end."""
    counter, draws = 0, 0
    taken = [0] * nunits
    k = [0] * grid
    active = list(range(grid))
    while active and draws <= nunits + grid:   # (a launch makes at most nunits + grid draws; a wrong ndraws may loop)
        i = rng.randrange(len(active))
        w = active[i]
        if k[w] < nstatic:
            t = w + k[w] * grid
        else:
            d = counter
            counter += 1
            draws += 1
            if d == ndraws - 1:
                counter = 0
            t = nstatic * grid + d
        k[w] += 1
        if t < nunits:
            taken[t] += 1
        elif k[w] >= nstatic:   # a bad ticket: the warp draws no more (a bad static ticket is followed by static ones only)
            active[i] = active[-1]
            active.pop()
    return draws, taken, counter


def schedule_cases():
    rng = random.Random(7)
    cases = [(1, 1, 85), (2, 1, 85), (1, 2, 0), (3, 8, 85), (5, 5, 100), (7, 3, 100), (1584, 1584, 85), (1585, 1584, 85), (4000, 1584, 85)]
    for _ in range(120):
        nunits = rng.choice([rng.randint(1, 40), rng.randint(1, 3000)])
        grid = rng.randint(1, nunits) if rng.random() < 0.85 else rng.randint(nunits, nunits + 50)
        pct = rng.choice([0, 50, 85, 100, rng.randint(0, 100)])
        cases.append((nunits, grid, pct))
    return cases


def test_ticket_schedule_draws_every_unit_once_and_resets_the_counter(lib):
    rng = random.Random(11)
    for nunits, grid, pct in schedule_cases():
        nstatic, ndraws = ctypes.c_uint32(), ctypes.c_uint32()
        lib.tickets(nunits, grid, pct, ctypes.byref(nstatic), ctypes.byref(ndraws))
        draws, taken, counter = simulate(nunits, grid, nstatic.value, ndraws.value, rng)
        case = (nunits, grid, pct, nstatic.value, ndraws.value)
        assert draws == ndraws.value, case
        assert all(n == 1 for n in taken), case
        assert counter == 0, case


# ---- kernel choice ---------------------------------------------------------------------------------------------------

W, H, PS = 64, 48, 64
BASE = dict(force_flat=0, have_plan=1, has_box=1, w=W, h=H, opx=1, out=0x200000, pitch=W, out_stride=W * H, faces=0x100000,
            face_stride=6 * PS * PS, nframes=2, rowbytes=0, origins=None)
ATLAS = [(c * PS, r * PS) for r in range(2) for c in range(3)]   # a 3x2 atlas, 16-byte aligned origins


def choose(lib, **kw):
    a = dict(BASE, **kw)
    org = a["origins"] or []
    arr = (ctypes.c_int32 * max(1, 2 * len(org)))(*[v for xy in org for v in xy])
    return lib.choose(a["force_flat"], a["have_plan"], a["has_box"], a["w"], a["h"], a["opx"], a["out"], a["pitch"], a["out_stride"], a["faces"],
                      a["face_stride"], a["nframes"], a["rowbytes"], ctypes.cast(arr, ctypes.c_void_p), len(org))


KERNEL_CASES = [
    ("dense 64x48 8-bit", {}, RING),
    ("odd x0 origin", dict(out=0x200001, pitch=W + 8), SCALAR),
    ("pitch not a multiple of 4 px", dict(pitch=W + 2), SCALAR),
    ("6x2 dense (W % 4 != 0, W*H % 4 == 0)", dict(w=6, h=2, pitch=6, out_stride=12), VECTOR),
    ("6x3 dense", dict(w=6, h=3, pitch=6, out_stride=20), SCALAR),
    ("RGBA origin 4- but not 16-byte aligned", dict(opx=4, out=0x200004, pitch=4 * W + 64, out_stride=(4 * W + 64) * H), SCALAR),
    ("RGBA dense", dict(opx=4, pitch=4 * W, out_stride=4 * W * H), RING),
    ("unaligned frame stride, 1 frame", dict(out_stride=W * H + 1, nframes=1), RING),
    ("unaligned frame stride, 2 frames", dict(out_stride=W * H + 1), SCALAR),
    ("faces 8-byte aligned, plan with BOX tiles", dict(faces=0x100008), VECTOR),
    ("faces 8-byte aligned, plan without BOX tiles", dict(faces=0x100008, has_box=0), RING),
    ("face stride % 16 != 0, 2 frames", dict(face_stride=6 * PS * PS + 8), VECTOR),
    ("face stride % 16 != 0, 1 frame", dict(face_stride=6 * PS * PS + 8, nframes=1), RING),
    ("layout rowbytes % 16 != 0", dict(rowbytes=3 * PS + 8, origins=ATLAS), VECTOR),
    ("layout origin x % 16 != 0", dict(rowbytes=3 * PS + 16, origins=ATLAS[:5] + [(2 * PS + 8, PS)]), VECTOR),
    ("layout with 16-aligned rowbytes and origins", dict(rowbytes=3 * PS + 16, origins=ATLAS), RING),
    ("blinky_set_kernel(1)", dict(force_flat=1), VECTOR),
    ("blinky_set_kernel(1), unaligned origin", dict(force_flat=1, out=0x200002), SCALAR),
    ("no plan (extent > 65536)", dict(have_plan=0), VECTOR),
]


@pytest.mark.parametrize("name,kw,expected", KERNEL_CASES, ids=[c[0] for c in KERNEL_CASES])
def test_kernel_choice(lib, name, kw, expected):
    assert choose(lib, **kw) == expected


# ---- frames per unit -------------------------------------------------------------------------------------------------

def test_frames_per_unit(lib):
    grid = 132 * 12
    assert lib.fpu(7900, 16, grid, 0) == 16
    assert lib.fpu(5000, 16, grid, 0) == 8
    for tiles in (1, 100, 5000, 7900, 100000):
        assert lib.fpu(tiles, 1, grid, 0) == 1
    assert lib.fpu(7900, 16, grid, 4) == 4      # BLINKY_FCHUNK
    assert lib.fpu(7900, 3, grid, 8) == 3       # ... clamped to nframes
    assert lib.fpu(7900, 40, grid, 32) == 32    # ... which may exceed 16
    for nframes in range(1, 40):
        assert 1 <= lib.fpu(3000, nframes, grid, 0) <= min(nframes, 16)


# ---- ring geometry ---------------------------------------------------------------------------------------------------

SMEM_H100 = 233472
FIXED_PLAIN = 6 * 8 + 16   # the ring kernel's barriers (kRingBarBytes)


def geometry(lib, smem, want, merged, fixed, max_box, override=0):
    warps, ring = ctypes.c_int(), ctypes.c_uint32()
    lib.geometry(smem, want, int(merged), fixed, max_box, override, ctypes.byref(warps), ctypes.byref(ring))
    return warps.value, ring.value


def test_ring_geometry_default_h100(lib):
    assert geometry(lib, SMEM_H100, 12, False, FIXED_PLAIN, 8192) == (12, 18304)
    assert geometry(lib, SMEM_H100, 12, True, FIXED_PLAIN, 8192) == (12, 15488)
    # small plans get at least 8 KB; BLINKY_RING_BYTES sets the ring, never below the largest box
    assert geometry(lib, SMEM_H100, 12, False, FIXED_PLAIN, 2176) == (12, 8192)
    assert geometry(lib, SMEM_H100, 12, False, FIXED_PLAIN, 8192, override=4000) == (12, 8192)
    assert geometry(lib, SMEM_H100, 12, False, FIXED_PLAIN, 2176, override=4000) == (12, 3968)
    assert geometry(lib, 8000, 4, False, FIXED_PLAIN, 8192) == (0, 0)


def fits(smem, warps, merged, fixed, max_box):
    return smem // (warps + 2 * merged) >= 1024 + fixed + max_box


def test_ring_geometry_invariants(lib):
    rng = random.Random(3)
    for _ in range(3000):
        smem = rng.randint(20000, 240000)
        want = rng.randint(1, 16)
        merged = rng.random() < 0.5
        fixed = FIXED_PLAIN + rng.choice([0, 1024, 1536, 2560])
        max_box = 128 * rng.randint(1, 128)
        override = rng.choice([0, 0, rng.randint(1, 40000)])
        warps, ring = geometry(lib, smem, want, merged, fixed, max_box, override)
        case = (smem, want, merged, fixed, max_box, override, warps, ring)
        if warps == 0:
            assert ring == 0 and not any(fits(smem, w, merged, fixed, max_box) for w in range(1, want + 1)), case
            continue
        assert 1 <= warps <= want, case
        assert ring % 128 == 0 and ring >= max_box, case
        assert (ring + fixed + 1024) * (warps + 2 * merged) <= smem, case
        assert not any(fits(smem, w, merged, fixed, max_box) for w in range(warps + 1, want + 1)), case


# ---- gather placement ------------------------------------------------------------------------------------------------

def test_gather_placement(lib):
    assert lib.items(10, 1) == 40 and lib.items(10, 4) == 40 and lib.items(10, 5) == 80
    assert lib.rides(10, 8, 4096, 0) == 1
    assert lib.rides(10, 9, 4096, 0) == 0     # more than kMergedFramesMax frames: K3 in front
    assert lib.rides(10, 1, 4096, 1) == 0     # BLINKY_SERIAL_GATHER
    assert lib.rides(0, 1, 4096, 0) == 0      # no GATHER tiles
    assert lib.rides(1024, 4, 4096, 0) == 1 and lib.rides(1025, 4, 4096, 0) == 0   # BLINKY_MERGED_ITEMS
    assert lib.rides(10, 1, 39, 0) == 0


# ---- kernel variant --------------------------------------------------------------------------------------------------

def test_kernel_variant_index_and_tags(lib):
    assert [lib.variant_index(i) for i in range(32)] == list(range(32))
    assert sum(lib.variant_exists(i) for i in range(32)) == 24
    assert all(lib.variant_exists(i) == (not (i & 8) or bool(i & 2)) for i in range(32))
    for i in range(32):
        want = (",keep=1" if i & 4 else "") + (",tables=1" if i & 8 else "") + (",layout=1" if i & 16 else "")
        assert lib.variant_tags(i).decode() == want
