// Decisions of the device warps (warp_device.cu): whether a call is accepted (check_warp), which kernel serves it, and
// how the ring kernel's launch is shaped — its geometry, where the GATHER tiles go, frames per unit and the ticket
// schedule.  Plain host arithmetic on the call, the context's state and the tile plan, no CUDA types, so that the CPU
// tests can pin it.
#pragma once

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <string>

#include "../../include/blinky_b200.h"
#include "face_layout.h"
#include "ray_warp.h"
#include "tile_plan.h"
#include "warp_device.h"

namespace blinky {

// The kernels' template flags for one warp.  Per-frame tables exist only in RGBA, so each kernel has 24 instances,
// one per index() that exists().
struct KernelVariant {
    bool rubix, rgba, keep, tables, layout;

    int index() const { return (rubix ? 1 : 0) | (rgba ? 2 : 0) | (keep ? 4 : 0) | (tables ? 8 : 0) | (layout ? 16 : 0); }
    static constexpr bool exists(int index) { return !(index & 8) || (index & 2); }
    // the flags in last_kernel, after rubix= and rgba=
    const char *tags() const {
        static const char *const kTags[8] = {"", ",keep=1", ",tables=1", ",keep=1,tables=1", ",layout=1", ",keep=1,layout=1",
                                             ",tables=1,layout=1", ",keep=1,tables=1,layout=1"};
        return kTags[index() >> 2];
    }
};

// The entry point's name: the prefix of its refusals ("warp" for internal calls; blinky_warp_host's have none).
inline const char *warp_entry_name(WarpEntry e) {
    static const char *const kNames[] = {"warp",
                                         "blinky_warp_device",
                                         "blinky_warp_device_rgba",
                                         "blinky_warp_device_view",
                                         "blinky_warp_device_view_rgba",
                                         "blinky_warp_device_view_rgba_tables",
                                         "blinky_warp_device_rays",
                                         "blinky_warp_device_rays_rgba",
                                         "blinky_warp_device_rays_supersampled",
                                         "blinky_warp_device_rays_bilinear",
                                         "blinky_warp_device_rays_trilinear",
                                         "blinky_ray_pyramid_bytes",
                                         ""};
    return kNames[static_cast<int>(e)];
}

// Whether the call r (with q, its rays, for the ray entry points) is accepted on state s: BLINKY_OK with what its
// launch needs in *c (a fresh CheckedWarp), or the BLINKY_E_* code of the first check it fails, with the reason in
// *why.  Each entry point keeps the order its checks have always had: the view entry points check the view rectangle
// before the lensmap, the dense ones after it, and the ray entry points check the state and their rays first.
// nframes <= 0 is accepted with nothing to launch once the checks before it pass.  Only a refusal builds a string.
inline int check_warp(const WarpRequest &r, const RayRequest &q, const WarpState &s, CheckedWarp *c, std::string *why) {
    const WarpEntry e = r.entry;
    const bool rays = e >= WarpEntry::Rays && e <= WarpEntry::RaysTrilinear;
    const bool view = e >= WarpEntry::View && e <= WarpEntry::RaysTrilinear;
    const bool host = e == WarpEntry::Host;
    const char *name = warp_entry_name(e);
    auto refuse = [why](int code, const char *prefix, const std::string &text) -> int {
        *why = *prefix ? std::string(prefix) + ": " + text : text;
        return code;
    };
    const int64_t W = s.width, H = s.height, ps = s.platesize, bpp = r.rgba ? 4 : 1;
    // the view: the rectangle at (x0, y0) of screens whose rows are rowbytes apart, or the whole screen
    const int64_t rowbytes = view || host ? r.rowbytes : W * bpp, x0 = r.x0, y0 = r.y0;
    auto check_view = [&]() -> int {
        if (!r.faces || !r.out) return refuse(BLINKY_E_INVALID, name, "NULL buffer");
        if (x0 < 0 || y0 < 0) return refuse(BLINKY_E_INVALID, name, "the view origin (x0, y0) must not be negative");
        if (rowbytes < (x0 + W) * bpp) return refuse(BLINKY_E_INVALID, name, std::string(host ? "dst_" : "") + "rowbytes too small for the view rectangle");
        if (view && r.nframes > 1 && static_cast<uint64_t>(r.out_stride) < static_cast<uint64_t>((y0 + H) * rowbytes))
            return refuse(BLINKY_E_INVALID, name, "screen_frame_stride too small for the view rectangle");
        if (r.rgba && ((reinterpret_cast<uintptr_t>(r.out) + static_cast<uintptr_t>(y0) * static_cast<uintptr_t>(rowbytes)) % 4 != 0 || rowbytes % 4 != 0 ||
                       (r.nframes > 1 && r.out_stride % 4 != 0)))
            return refuse(BLINKY_E_INVALID, name, "the RGBA view origin, rowbytes and screen_frame_stride must be 4-byte aligned");
        if (r.tables || e == WarpEntry::ViewRgbaTables) {
            // (16 bytes: the ring kernel restages a frame's table with 128-bit loads)
            if (!r.tables || reinterpret_cast<uintptr_t>(r.tables) % 16 != 0)
                return refuse(BLINKY_E_INVALID, name, "d_tables must be a non-NULL, 16-byte aligned device pointer");
            if (r.table_stride != 0 && (r.table_stride < 256 * sizeof(uint32_t) || r.table_stride % 16 != 0 || r.table_stride / 4 > UINT32_MAX))
                return refuse(BLINKY_E_INVALID, name, "table_stride must be 0 (one table for every frame) or at least 1024, a multiple of 16 and below 16 GB");
        }
        return BLINKY_OK;
    };
    // (the ray warps check it first, with their own code and text)
    auto check_installed = [&]() -> int {
        if (W > 0) return BLINKY_OK;
        if (rays) return refuse(BLINKY_E_STATE, name, "no lensmap installed (the view's size and background are the installed lensmap's)");
        if (e == WarpEntry::PyramidBytes) return refuse(BLINKY_E_STATE, name, "no lensmap installed (its plate size sizes the pyramid)");
        return refuse(BLINKY_E_CUDA, host ? "warp_host" : "warp", "no lensmap on the device (call blinky_build_lensmap)");
    };
    auto check_frames = [&]() -> int {
        return r.nframes > 65535 ? refuse(BLINKY_E_INVALID, rays ? name : "warp", "at most 65535 frames per launch") : BLINKY_OK;
    };
    // (the ray kernels pack a texel's px and py into 13 bits each: set_raymap's own limit, 6 * ps^2 < 2^28, keeps ps <= 6688)
    const bool ps_fits = ps * ps * kLayoutPlates <= 0x0FFFFFFF;
    auto pyramid_levels = [&]() { return c->lmax = ray_pyramid_levels(static_cast<int>(ps), s.globe.plates, c->level_size, c->level_off, &c->pyramid_bytes); };

    if (rays || e == WarpEntry::PyramidBytes) {
        if (const int rc = check_installed()) return rc;
        if (!s.globe.valid) return refuse(BLINKY_E_STATE, name, "no valid globe");
    }
    if (e == WarpEntry::PyramidBytes)
        return ps_fits && pyramid_levels() >= 0 ? BLINKY_OK
                                                : refuse(BLINKY_E_STATE, name, "the installed lensmap's plate size " + std::to_string(ps) +
                                                                                   " is beyond what the ray warps take (6 * platesize^2 must fit the 28-bit texel index)");
    if (rays) {
        if (s.globe.plate_script)
            return refuse(BLINKY_E_STATE, name, "the globe picks its plates with a globe_plate script, whose decisions can need the interpreter: "
                                                "map such rays with blinky_set_raymap_device and warp the installed lensmap");
        if (!q.rays) return refuse(BLINKY_E_INVALID, name, "NULL rays");
        if (reinterpret_cast<uintptr_t>(q.rays) % 4 != 0 || reinterpret_cast<uintptr_t>(q.xforms) % 4 != 0)
            return refuse(BLINKY_E_INVALID, name, "d_rays and d_xforms must be 4-byte aligned");
        // the entry points that take a factor (the supersampled factor 1 is blinky_warp_device_rays_rgba; the
        // bilinear one is a sample per pixel); the others' is 1
        const bool factored = e == WarpEntry::RaysSupersampled || e == WarpEntry::RaysBilinear;
        if (factored && (q.factor < (e == WarpEntry::RaysBilinear ? 1 : 2) || q.factor > 4))
            return refuse(BLINKY_E_INVALID, name, e == WarpEntry::RaysBilinear ? "factor must be 1, 2, 3 or 4" : "factor must be 2, 3 or 4");
        if (q.ray_stride != 0 &&
            (q.ray_stride < 12 * static_cast<size_t>(q.factor * q.factor) * static_cast<size_t>(W) * static_cast<size_t>(H) || q.ray_stride % 4 != 0))
            return refuse(BLINKY_E_INVALID, name, std::string("ray_stride must be 0 (one field for every frame) or a multiple of 4 of at least 12 * ") +
                                                      (factored ? "factor^2 * " : "") + "width * height");
        if (q.xform_stride != 0 && (q.xform_stride < 36 || q.xform_stride % 4 != 0))
            return refuse(BLINKY_E_INVALID, name, "xform_stride must be 0 (one matrix for every frame) or a multiple of 4 of at least 36");
        if (const int rc = check_frames()) return rc;
    }
    if (view || host)
        if (const int rc = check_view()) return rc;
    if (const int rc = check_installed()) return rc;
    c->launch = r.nframes > 0;
    if (!c->launch && !host) return BLINKY_OK;   // (blinky_warp_host checks its face layout first)
    if (!rays && !host) {
        if (const int rc = check_frames()) return rc;
        if (const int rc = check_view()) return rc;
    }
    if (rays) {
        if (!ps_fits)
            return refuse(BLINKY_E_STATE, "warp_rays", "the installed lensmap's plate size " + std::to_string(ps) +
                                                           " is beyond what a ray map takes (6 * platesize^2 must fit the 28-bit texel index)");
        // (the supersampled, bilinear and trilinear kernels index the field's pixels in 31 bits)
        const uint64_t field_pixels = static_cast<uint64_t>(q.factor) * q.factor * static_cast<uint64_t>(W) * static_cast<uint64_t>(H);
        if ((q.factor > 1 || q.filter != RayFilter::Nearest) && field_pixels > 0x7FFFFFFFu)
            return refuse(BLINKY_E_INVALID, "warp_rays", "a field of factor^2 * width * height = " + std::to_string(field_pixels) +
                                                             " pixels is beyond the kernel's 31-bit pixel index");
        // (the trilinear warp's pyramids: every plate of the globe, at the installed plate size)
        if (q.filter == RayFilter::Trilinear) {
            pyramid_levels();
            if (c->pyramid_bytes > 0 && !q.scratch)
                return refuse(BLINKY_E_INVALID, "warp_rays", "NULL scratch (the frames' pyramids need " + std::to_string(c->pyramid_bytes) + " bytes each)");
            if (reinterpret_cast<uintptr_t>(q.scratch) % 16 != 0) return refuse(BLINKY_E_INVALID, "warp_rays", "the scratch must be 16-byte aligned");
            if (static_cast<uint64_t>(q.scratch_bytes) < static_cast<uint64_t>(r.nframes) * c->pyramid_bytes)
                return refuse(BLINKY_E_INVALID, "warp_rays", "scratch_bytes " + std::to_string(q.scratch_bytes) + " is below nframes * " +
                                                                 std::to_string(c->pyramid_bytes) + " (blinky_ray_pyramid_bytes)");
        }
    }
    c->pitch = static_cast<size_t>(rowbytes);
    if (!host && c->pitch > (size_t{1} << 26))   // (the kernels step 32 rows in 32-bit offsets)
        return refuse(BLINKY_E_INVALID, "warp", "the output row pitch must hold a row of the view and be at most 64 MB");
    c->view = r.view(c->pitch);
    // The face layout against the installed lensmap (the plate size and the plates it samples change with every
    // build): a ray warp may sample any plate of the globe, the others the plates the lensmap samples.
    c->use_layout = rays || (s.layout_rowbytes > 0 && !r.dense_faces);
    if (s.layout_rowbytes > 0 && !r.dense_faces) {
        const uint64_t rb = static_cast<uint64_t>(s.layout_rowbytes), ups = static_cast<uint64_t>(ps);
        uint64_t rows = 0;
        for (int pl = 0; pl < s.layout_plates; ++pl) {
            const uint64_t x = static_cast<uint64_t>(s.layout_origins[2 * pl]), y = static_cast<uint64_t>(s.layout_origins[2 * pl + 1]);
            if (x + ups > rb)
                return refuse(BLINKY_E_INVALID, "face layout", "plate " + std::to_string(pl) + " at x = " + std::to_string(x) + " does not fit rowbytes " +
                                                                   std::to_string(rb) + " with plate size " + std::to_string(ups));
            rows = std::max(rows, y + ups);
            c->layout.plate_base[pl] = y * rb + x;
            c->layout.org_x[pl] = static_cast<int32_t>(x);
            c->layout.org_y[pl] = static_cast<int32_t>(y);
        }
        for (int pl = s.layout_plates; pl < kLayoutPlates; ++pl) {
            const int *rc = s.plate_rect[pl];
            if (rays ? pl < s.globe.plates : s.display[pl] || (rc[0] <= rc[2] && rc[1] <= rc[3]))
                return refuse(BLINKY_E_INVALID, "face layout", std::string(rays ? "the globe has plate " : "the lensmap samples plate ") + std::to_string(pl) +
                                                                   ", which has no origin (the layout has " + std::to_string(s.layout_plates) + ")");
        }
        if (r.nframes > 1 && static_cast<uint64_t>(r.face_stride) < rows * rb)
            return refuse(BLINKY_E_INVALID, "face layout", "face_stride " + std::to_string(r.face_stride) + " is smaller than a frame's surface (" +
                                                               std::to_string(rows) + " rows of " + std::to_string(rb) + " bytes)");
        c->layout.rowbytes = static_cast<uint32_t>(rb);
        c->layout.ps = static_cast<uint32_t>(ups);
        c->layout.ps2 = static_cast<uint32_t>(ups * ups);
        c->layout.div_ps = make_fastdiv(c->layout.ps);
        c->layout.div_ps2 = make_fastdiv(c->layout.ps2);
        c->layout_rows = static_cast<uint32_t>(rows);
    } else if (rays) {   // dense [plate][ps][ps] frames: the layout with rowbytes = ps
        for (int i = 0; i < kLayoutPlates; ++i) c->layout.plate_base[i] = static_cast<uint64_t>(i) * static_cast<uint64_t>(ps * ps);
        c->layout.rowbytes = static_cast<uint32_t>(ps);
    }
    return BLINKY_OK;
}

enum class WarpKernel { Ring, Vector, Scalar };   // warp_ring_kernel (with K3), K1 warp_gather_kernel, K0 warp_scalar_kernel

// r with its bytes between output rows `pitch` (never 0) and the face layout it reads (nullptr: dense frames), on the
// view and tile plan in place; force_flat: blinky_set_kernel(BLINKY_KERNEL_GATHER).
inline WarpKernel choose_kernel(const WarpRequest &r, size_t pitch, const FaceLayoutParams *layout, int width, int height, bool have_plan,
                                bool plan_has_box, bool force_flat) {
    const size_t opx = r.rgba ? 4 : 1, word = 4 * opx;   // 4-pixel words: the ring kernel's and K1's stores
    const bool frames_aligned = reinterpret_cast<uintptr_t>(r.view(pitch)) % word == 0 && (r.out_stride % word == 0 || r.nframes == 1);
    // the ring kernel: W % 4 == 0 and the view's origin, pitch and frame stride aligned to 4 pixels; TMA boxes need
    // 16-byte aligned faces and frame stride, and with a face layout 16-byte aligned rows and plate x origins
    bool ring = !force_flat && have_plan && width % 4 == 0 && pitch % word == 0 && frames_aligned &&
                (!plan_has_box || (reinterpret_cast<uintptr_t>(r.faces) % 16 == 0 && (r.face_stride % 16 == 0 || r.nframes == 1)));
    if (layout) {
        ring = ring && layout->rowbytes % 16 == 0;
        for (const int32_t x : layout->org_x) ring = ring && x % 16 == 0;   // (plates without an origin: 0)
    }
    if (ring) return WarpKernel::Ring;
    // K1: dense frames need W*H % 4 == 0, pitched ones W % 4 == 0 (no quad straddles two rows)
    const bool pitched = pitch != static_cast<size_t>(width) * opx;
    const size_t npix = static_cast<size_t>(width) * static_cast<size_t>(height);
    const bool vector = (pitched ? width % 4 == 0 && pitch % word == 0 : npix % 4 == 0) && frames_aligned;
    return vector ? WarpKernel::Vector : WarpKernel::Scalar;
}

// The warp from a ray field (ray_warp_kernel): one thread per 4-pixel quad of a row, written as one word, when W % 4
// == 0 and the view's origin, pitch and frame stride allow 4-pixel words; otherwise one thread per pixel.
inline bool ray_warp_quads(const WarpRequest &r, size_t pitch, int width) {
    const size_t word = 4 * (r.rgba ? 4 : 1);
    const bool frames_aligned = reinterpret_cast<uintptr_t>(r.view(pitch)) % word == 0 && (r.out_stride % word == 0 || r.nframes == 1);
    return width % 4 == 0 && pitch % word == 0 && frames_aligned;
}

// Frames each thread of a ray warp carries.  With one ray field for every frame (ray_stride 0) a thread carries several,
// so that the field is read once per launch rather than once per frame — but no more than leaves the launch at least
// `resident_threads` threads (what the GPU holds at once: SMs x threads per SM), so that a small view in a large batch
// does not leave most SMs idle.  nitems: threads per frame (quads or pixels).  Per-frame fields: one frame per thread.
inline int ray_warp_frames_per_thread(size_t ray_stride, int nframes, uint32_t nitems, uint32_t resident_threads) {
    if (ray_stride != 0 || nframes <= 1) return 1;
    const uint64_t want = (static_cast<uint64_t>(resident_threads) + std::max<uint32_t>(nitems, 1u) - 1) / std::max<uint32_t>(nitems, 1u);
    const uint64_t splits = std::min<uint64_t>(static_cast<uint64_t>(nframes), std::max<uint64_t>(want, 1u));
    return static_cast<int>(static_cast<uint64_t>(nframes) / splits);   // (rounded down: at least `splits` rows of threads)
}

// The launch shape of the ray warp q of r into a view of width x height: quads only for the nearest filter at factor 1
// (every other filter writes one RGBA pixel per thread), frames per thread for that item count, and a grid that covers
// every item and every frame.
inline RayWarpShape ray_warp_shape(const WarpRequest &r, const RayRequest &q, size_t pitch, int width, int height, uint32_t resident_threads) {
    RayWarpShape s;
    s.quads = q.filter == RayFilter::Nearest && q.factor == 1 && ray_warp_quads(r, pitch, width);
    const size_t npix = static_cast<size_t>(width) * static_cast<size_t>(height);
    s.nitems = static_cast<uint32_t>(s.quads ? npix / 4 : npix);
    s.frames_per_thread = ray_warp_frames_per_thread(q.ray_stride, r.nframes, s.nitems, resident_threads);
    s.grid_x = (s.nitems + kRayThreads - 1) / kRayThreads;
    s.grid_y = static_cast<uint32_t>((r.nframes + s.frames_per_thread - 1) / s.frames_per_thread);
    return s;
}

struct RingGeometry {
    int warps;            // resident ring warps per SM; 0: the plan's largest box does not fit a ring
    uint32_t ring_bytes;  // each warp's staging ring (a multiple of 128)
};

// As many warps per SM as `want`, each with the largest staging ring that still lets them — plus two gather CTAs,
// which carry the same allocation, when GATHER tiles ride along — share the SM's shared memory (1024 bytes per CTA
// of it are the system's, `fixed` the kernel's barriers and tables); fewer warps if the plan's largest box would
// not fit such a ring.  The ring holds two of the plan's largest boxes and an entry block (two boxes of any size and
// the next unit's entries in flight), at least 8 KB; ring_bytes_override > 0 (BLINKY_RING_BYTES) sets it instead.
inline RingGeometry ring_geometry(size_t smem_per_sm, int want, bool merged_gather, size_t fixed, uint32_t max_box, int ring_bytes_override) {
    for (; want >= 1; --want) {
        const size_t per_cta = smem_per_sm / static_cast<size_t>(want + (merged_gather ? 2 : 0));
        if (per_cta < 1024 + fixed + max_box) continue;
        const uint32_t room = static_cast<uint32_t>((per_cta - 1024 - fixed) / 128 * 128);
        uint32_t ring_bytes = std::min(room, std::max(2u * max_box + kBoxBlockBytes, 8192u));
        if (ring_bytes_override > 0) ring_bytes = std::min(room, std::max<uint32_t>(max_box, static_cast<uint32_t>(ring_bytes_override) / 128 * 128));
        return {want, ring_bytes};
    }
    return {0, 0};
}

// A gather item is one GATHER tile's kGatherRows rows in kGatherFrames frames: one gather CTA of the ring kernel's
// launch (gather_item).
constexpr int kGatherRows = 8, kGatherFrames = 4;
constexpr int kMergedFramesMax = 8;

inline uint32_t gather_items(uint32_t ngather_tiles, int nframes) {
    return ngather_tiles * (kTileH / kGatherRows) * static_cast<uint32_t>((nframes + kGatherFrames - 1) / kGatherFrames);
}

// GATHER tiles ride in the ring kernel's launch only in launches of at most kMergedFramesMax frames with at most
// merged_items_max gather items (BLINKY_MERGED_ITEMS), where a second kernel launch costs more than they do;
// otherwise, or with serial_gather (BLINKY_SERIAL_GATHER), the gather kernel K3 goes in front.  Measured on the H100
// (80GB HBM3, 400 W): riding along is 2-20 % faster for 1-8 frames of 4K panini and trism, but with 16 frames K3 in
// front is faster by 1.5-10 % (panini, stereographic, trism, 1080p panini; the 1080p batch prefers K3 from 8 frames
// on, by 10 %, and keeps riding along there).
inline bool gather_rides_along(uint32_t ngather_tiles, int nframes, int merged_items_max, bool serial_gather) {
    return !serial_gather && ngather_tiles > 0 && nframes <= kMergedFramesMax &&
           gather_items(ngather_tiles, nframes) <= static_cast<uint32_t>(merged_items_max);
}

// A unit pays a fixed cost (entry unpack, ring refill across the boundary: ~kUnitCost frame times) and the launch
// ends with a tail of about one unit: the chunk of 1..16 frames that minimises units-per-warp x (chunk + kUnitCost) +
// chunk.  kUnitCost = 2 fits the H100 (80GB HBM3, 400 W): 16-frame units beat 8-frame ones by 4-7 % on the 4K
// batches of ~7900 ring tiles (panini, stereographic, quincuncial, trism), and lose 1-3 % on those of ~5000 (hammer,
// fisheye1), which keep 8.  fchunk_override > 0 (BLINKY_FCHUNK) sets the chunk; never more than nframes.
constexpr double kUnitCost = 2.0;

inline uint32_t frames_per_unit(uint32_t ring_tiles, uint32_t nframes, uint32_t grid, int fchunk_override) {
    if (fchunk_override > 0) return std::min(static_cast<uint32_t>(fchunk_override), nframes);
    uint32_t fchunk = 1;
    double best = 0;
    for (uint32_t c = 1; c <= std::min<uint32_t>(nframes, 16u); ++c) {
        const double units = static_cast<double>(ring_tiles) * ((nframes + c - 1) / c);
        const double cost = std::max(1.0, units / grid) * (c + kUnitCost) + c;
        if (c == 1 || cost < best) best = cost, fchunk = c;
    }
    return std::min(fchunk, nframes);
}

struct TicketSchedule {
    uint32_t nstatic;   // units per warp assigned statically (warp w owns w, w + grid, ...)
    uint32_t ndraws;    // counter draws the launch makes
};

// static_pct percent of the units are static, in whole rounds of `grid` warps (grid >= 1).  Every unit beyond the
// static ones is drawn exactly once, and every warp that draws at all draws exactly one ticket past the end (it
// stops at its first bad ticket).  A warp draws iff its last static ticket is good (all warps when there are no
// static rounds).  The kernel's counter returns to 0 only if ndraws is exact (ticket_drawn).
inline TicketSchedule ticket_schedule(uint32_t nunits, uint32_t grid, int static_pct) {
    const uint32_t nstatic = static_cast<uint32_t>(static_cast<uint64_t>(nunits) * static_cast<uint64_t>(static_pct) / 100u / grid);
    const uint64_t nst = static_cast<uint64_t>(nstatic) * grid;
    const uint32_t good = nunits > nst ? static_cast<uint32_t>(nunits - nst) : 0u;
    uint32_t drawers = grid;
    if (nstatic > 0) {
        const uint64_t before_last = static_cast<uint64_t>(nstatic - 1) * grid;
        drawers = nunits > before_last ? static_cast<uint32_t>(std::min<uint64_t>(nunits - before_last, grid)) : 0u;
    }
    return {nstatic, good + drawers};
}

}  // namespace blinky
