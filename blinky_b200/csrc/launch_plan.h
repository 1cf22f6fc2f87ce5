// Launch decisions of the device warps (warp_device.cu): which kernel serves a call, and how the ring kernel's
// launch is shaped — its geometry, where the GATHER tiles go, frames per unit and the ticket schedule.  Plain host
// arithmetic on the call and the tile plan, no CUDA types, so that the CPU tests can pin it.
#pragma once

#include <algorithm>
#include <cstddef>
#include <cstdint>

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

enum class WarpKernel { Ring, Vector, Scalar };   // warp_ring_kernel (with K3), K1 warp_gather_kernel, K0 warp_scalar_kernel

// r with its bytes between output rows `pitch` (never 0) and the face layout it reads (nullptr: dense frames), on the
// view and tile plan in place; force_flat: blinky_set_kernel(BLINKY_KERNEL_GATHER).
inline WarpKernel choose_kernel(const WarpRequest &r, size_t pitch, const FaceLayoutParams *layout, int width, int height, bool have_plan,
                                bool plan_has_box, bool force_flat) {
    const size_t opx = r.rgba ? 4 : 1, word = 4 * opx;   // 4-pixel words: the ring kernel's and K1's stores
    const bool frames_aligned = reinterpret_cast<uintptr_t>(r.out) % word == 0 && (r.out_stride % word == 0 || r.nframes == 1);
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
    const bool frames_aligned = reinterpret_cast<uintptr_t>(r.out) % word == 0 && (r.out_stride % word == 0 || r.nframes == 1);
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
