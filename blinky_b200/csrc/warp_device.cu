// Device side of the H100 lens-warp path — kernels, resident state, frame pipeline.
//
// The reference's hot loop (the reference's engine/NQ/fisheye.c:2406-2424) is,
// per screen pixel: load an 8-byte pointer, load the source byte through it,
// optionally map it through a 256-entry tint LUT chosen by a second per-pixel
// byte, store one byte.  Here one packed 32-bit lensmap entry per pixel
// replaces pointer + tint byte (4 B instead of 9 B read per pixel), entries
// are fetched as 128-bit vectors, source bytes are gathered through the
// read-only path, and four output pixels are written per 32-bit store so that
// every warp-level store instruction covers one full 128-byte line.
//
// sm_90a only.  HBM-bound byte work: no tensor cores on purpose.
#include "warp_device.h"

#include <cuda.h>  // CUtensorMap types only; the driver entry point is fetched at run time
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

#include "../../include/blinky_b200.h"
#include "face_layout.h"
#include "launch_plan.h"
#include "lens_device.h"
#include "ray_warp.h"
#include "tile_plan.h"
#include "tile_plan_device.h"

namespace blinky {

namespace {

constexpr int kThreads = 256;
constexpr int kChunks = 4;                            // quads (4-pixel groups) per thread
constexpr int kQuadsPerBlock = kThreads * kChunks;    // 1024 quads = 4096 pixels per CTA
constexpr int kPixelsPerBlock = kQuadsPerBlock * 4;

struct WarpParams {
    const uint4 *lensmap4;      // packed entries, 4 per element; padded to whole CTAs
    const uint8_t *faces;       // frame 0
    size_t face_stride;         // bytes between frames
    const uint32_t *bg32;       // background, 4 pixels per element (padded like the lensmap)
    const uint8_t *lut;         // [6][256] rubix tint LUTs
    const uint32_t *rgba;       // [256] palette expansion table (RGBA mode); TABLES: frame 0's
    void *out;                  // view origin of frame 0
    size_t out_stride;          // bytes between frames
    uint32_t nquads;            // ceil(W*H / 4)
    uint32_t npix;              // W*H
    uint32_t width;             // W
    uint32_t out_pitch;         // bytes between output rows
    bool pitched;               // out_pitch != W * bytes per pixel: rows are addressed one by one
    uint32_t table_words;       // TABLES: words between the tables of consecutive frames
};

__device__ __forceinline__ uint4 ld_lensmap(const uint4 *p) {
    // streamed once per frame by this SM: keep it out of L1 so the gathers own L1
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t ld_face(const uint8_t *p) {
    // read-only path, allocate in L1: neighbouring pixels hit the same sectors
    uint32_t v;
    asm volatile("ld.global.nc.u8 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

__device__ __forceinline__ void st_stream_u32(uint32_t *p, uint32_t v) {
    asm volatile("st.global.cs.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ void st_stream_v4(uint4 *p, uint4 v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ void st_stream_u8(uint8_t *p, uint32_t v) {
    asm volatile("st.global.cs.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// keep_unmapped: the mapped pixels of a partly mapped quad, one store each (a byte, or an RGBA word), so the
// caller's other pixels are never read or rewritten — another writer may own them (neighbouring view rectangles
// of one screen, warped concurrently).  px: the four output values, valid4: bit k = pixel k is mapped.
template <bool RGBA>
__device__ __forceinline__ void st_quad_masked(uint8_t *dst, const uint32_t (&px)[4], uint32_t valid4) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (!((valid4 >> k) & 1u)) continue;
        if (RGBA) st_stream_u32(reinterpret_cast<uint32_t *>(dst + 4 * k), px[k]);
        else st_stream_u8(dst + k, px[k]);
    }
}

// byte offset of pixel `pix` (dense index y*W + x) in a frame of the output
__device__ __forceinline__ size_t out_offset(const WarpParams &p, uint32_t pix, uint32_t opx) {
    if (!p.pitched) return static_cast<size_t>(pix) * opx;
    const uint32_t y = pix / p.width;
    return static_cast<size_t>(y) * p.out_pitch + static_cast<size_t>(pix - y * p.width) * opx;
}

// --------------------------------------------------------------------------
// K1: direct gather.  grid = (ceil(nquads/1024), nframes), block = 256.
// Thread t of CTA b owns quads b*1024 + c*256 + t, c = 0..3, so each of the
// four 128-bit lensmap loads of a warp covers 512 contiguous bytes and each
// 32-bit output store of a warp covers 128 contiguous bytes.  A pitched output
// needs W % 4 == 0, so that no quad straddles two rows.
// KEEP (keep_unmapped): unmapped pixels are not written and the background is
// never read; a partly mapped quad is stored pixel by pixel.
// TABLES (RGBA only): frame f is expanded through its own table at
// p.rgba + f * p.table_words, in every kernel below.
// LAYOUT: the faces follow a face layout (face_layout.h): a texel's address is
// its plate-space offset split by layout_texel, in every kernel below.  The
// layout is the kernels' last parameter, which the dense instances never read.
// --------------------------------------------------------------------------
template <bool RUBIX, bool RGBA, bool KEEP, bool TABLES, bool LAYOUT>
__global__ void __launch_bounds__(kThreads) warp_gather_kernel(const WarpParams p, const __grid_constant__ FaceLayoutParams lay) {
    __shared__ uint8_t s_lut[RUBIX ? 6 * 256 : 4];
    __shared__ uint32_t s_rgba[RGBA ? 256 : 1];
    if (RUBIX) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.lut);
        uint32_t *dst = reinterpret_cast<uint32_t *>(s_lut);
        for (int i = threadIdx.x; i < 6 * 256 / 4; i += kThreads) dst[i] = __ldg(src + i);
    }
    if (RGBA) {
        // (one frame per CTA: its table)
        const uint32_t *table = TABLES ? p.rgba + static_cast<size_t>(blockIdx.y) * p.table_words : p.rgba;
        for (int i = threadIdx.x; i < 256; i += kThreads) s_rgba[i] = __ldg(table + i);
    }
    if (RUBIX || RGBA) __syncthreads();

    const uint8_t *__restrict__ faces = p.faces + static_cast<size_t>(blockIdx.y) * p.face_stride;
    const uint32_t q0 = blockIdx.x * kQuadsPerBlock + threadIdx.x;

    uint4 e[kChunks];
#pragma unroll
    for (int c = 0; c < kChunks; ++c) e[c] = ld_lensmap(p.lensmap4 + q0 + c * kThreads);  // padded: always in range

    uint32_t v[kChunks][4];
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
        const uint32_t ent[4] = {e[c].x, e[c].y, e[c].z, e[c].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            v[c][k] = 0;
            if (ent[k] & BLINKY_LM_VALID)
                v[c][k] = ld_face(LAYOUT ? faces + layout_texel(ent[k] & BLINKY_LM_INDEX_MASK, lay) : faces + (ent[k] & BLINKY_LM_INDEX_MASK));
        }
    }

#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
        const uint32_t q = q0 + c * kThreads;
        if (q >= p.nquads) continue;
        const uint32_t ent[4] = {e[c].x, e[c].y, e[c].z, e[c].w};
        const uint32_t all_valid = ent[0] & ent[1] & ent[2] & ent[3] & BLINKY_LM_VALID;
        const uint32_t valid4 = (ent[0] >> 31) | ((ent[1] >> 31) << 1) | ((ent[2] >> 31) << 2) | ((ent[3] >> 31) << 3);
        if (KEEP && valid4 == 0) continue;
        uint32_t bgw = 0;
        if (!KEEP && !all_valid) bgw = __ldg(p.bg32 + q);
        uint32_t px[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint32_t b = v[c][k];
            if (RUBIX) {
                const uint32_t t = (ent[k] >> BLINKY_LM_TINT_SHIFT) & 7u;
                if (t != BLINKY_LM_TINT_NONE) b = s_lut[t * 256 + b];
            }
            if (!(ent[k] & BLINKY_LM_VALID)) b = (bgw >> (8 * k)) & 0xffu;
            px[k] = b;
        }
        uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(blockIdx.y) * p.out_stride + out_offset(p, 4 * q, RGBA ? 4 : 1);
        if (RGBA) {
#pragma unroll
            for (int k = 0; k < 4; ++k) px[k] = s_rgba[px[k]];
        }
        if (KEEP && !all_valid) {
            st_quad_masked<RGBA>(o, px, valid4);
        } else if (RGBA) {
            st_stream_v4(reinterpret_cast<uint4 *>(o), make_uint4(px[0], px[1], px[2], px[3]));
        } else {
            st_stream_u32(reinterpret_cast<uint32_t *>(o), px[0] | (px[1] << 8) | (px[2] << 16) | (px[3] << 24));
        }
    }
}

// --------------------------------------------------------------------------
// K0: scalar kernel, one pixel per thread, byte stores.  Used only when the
// frame size or the caller's pointers rule out 32-bit stores (W*H % 4 != 0,
// unaligned strides, or a view rectangle whose origin or pitch is not a
// multiple of 4 pixels) — a correctness path for ragged sizes, not a fast path.
// --------------------------------------------------------------------------
template <bool RUBIX, bool RGBA, bool KEEP, bool TABLES, bool LAYOUT>
__global__ void __launch_bounds__(kThreads) warp_scalar_kernel(const WarpParams p, const __grid_constant__ FaceLayoutParams lay) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= p.npix) return;
    const uint32_t ent = __ldg(reinterpret_cast<const uint32_t *>(p.lensmap4) + i);
    if (KEEP && !(ent & BLINKY_LM_VALID)) return;
    const uint8_t *faces = p.faces + static_cast<size_t>(blockIdx.y) * p.face_stride;
    uint32_t b;
    if (ent & BLINKY_LM_VALID) {
        b = ld_face(LAYOUT ? faces + layout_texel(ent & BLINKY_LM_INDEX_MASK, lay) : faces + (ent & BLINKY_LM_INDEX_MASK));
        if (RUBIX) {
            const uint32_t t = (ent >> BLINKY_LM_TINT_SHIFT) & 7u;
            if (t != BLINKY_LM_TINT_NONE) b = __ldg(p.lut + t * 256 + b);
        }
    } else {
        b = __ldg(reinterpret_cast<const uint8_t *>(p.bg32) + i);
    }
    uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(blockIdx.y) * p.out_stride + out_offset(p, i, RGBA ? 4 : 1);
    if (RGBA) *reinterpret_cast<uint32_t *>(o) = __ldg((TABLES ? p.rgba + static_cast<size_t>(blockIdx.y) * p.table_words : p.rgba) + b);
    else *o = static_cast<uint8_t>(b);
}


// --------------------------------------------------------------------------
// K2: ring kernel.  Every WARP is its own pipeline (one warp per CTA, 12 resident per SM): it
// takes work units (tile, chunk of frames) — most from a static schedule, the tail from a ticket
// counter —, keeps the tile's lensmap entries in REGISTERS for all frames of the unit, and feeds
// itself through a private ring of TMA tensor loads:
//   * the ring is a byte FIFO of items in shared memory: per unit its entry block (2 KB of 16-bit
//     offsets, bulk copy cp.async.bulk) and then one source box per frame (ONE 4-D TMA tensor
//     load: x, y, plate, frame), each completing on its own mbarrier, issued by lane 0 from a
//     cursor that runs up to three units ahead.
//   * per unit: the lane reads its 32 entries out of the ring with four 128-bit shared loads and
//     unpacks them once.
//   * per frame: the warp waits for the box, does 32 byte loads from shared memory per lane (one
//     per output pixel), packs them with PRMT into eight 32-bit words, issues the next item(s) of
//     its sequence as soon as the consumed bytes sit in registers, and writes the words with
//     streaming stores.
// There is no producer warp, no cross-warp barrier, no per-pixel entry traffic per frame, and no
// global load on a scoreboard in the frame loop.  More warps or deeper rings lose as much L2
// locality on the halo sectors neighbouring tiles share as they gain latency hiding.
// EMPTY tiles copy the background.  GATHER tiles (plate seams, singular points, boxes too large to
// stage) are not the ring warps': see gather_item.
// --------------------------------------------------------------------------
constexpr int kRingBoxes = 6;                                 // items (boxes, entry blocks) in flight per warp at most (one mbarrier each)
constexpr int kRingBarBytes = kRingBoxes * 8 + 16;            // mbarriers, padded to a multiple of 16 bytes
static_assert(kRingBarBytes % 16 == 0 && kBoxBlockBytes % 128 == 0, "ring items are multiples of 128 bytes (TMA destinations), entry blocks are read with 128-bit loads");

struct RingParams {
    const TileDesc *tiles;
    const uint8_t *entries;
    const uint8_t *faces;
    size_t face_stride;
    const uint8_t *bg;
    const uint8_t *lut;
    const uint32_t *rgba;
    void *out;              // view origin of frame 0
    size_t out_stride;      // bytes between frames
    uint32_t out_pitch;     // PIXELS between output rows (the background and the lensmap stay dense: W per row)
    uint32_t *ticket;       // work counter: 0 when the launch starts, set back to 0 by its last draw (see ticket_drawn)
    uint32_t ndraws;        // counter draws the launch makes (see launch_ring)
    uint32_t nstatic;       // units per warp that are assigned statically (warp w owns w, w+NW, ...) before it draws tickets
    uint32_t nbox, ngather, ntiles;
    uint32_t nframes, fchunk, nchunks, nunits;
    uint32_t ring_bytes;    // the warp's staging ring: boxes are packed into it one behind the other (multiple of 128)
    uint32_t max_inflight;  // boxes a warp keeps in flight at most (<= kRingBoxes)
    uint32_t ring_grid;     // CTAs [0, ring_grid) are ring warps, the CTAs behind them take one gather item each
    int width, height;
    uint32_t zero;  // always 0, but only the host knows: see stage_dep()
    uint32_t table_words;   // TABLES: words between the RGBA tables of consecutive frames (rgba: frame 0's)
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
// NB (scripts/tma_probe.cu): the innermost coordinate must be a
// multiple of 16 bytes or the TMA unit raises "illegal instruction".
__device__ __forceinline__ void tma_load_box(uint32_t smem_dst, const CUtensorMap *tmap, int x, int y, int plate, int frame, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(smem_dst), "l"(tmap), "r"(x), "r"(y), "r"(plate), "r"(frame), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t addr) {
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
    return r;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

__device__ __forceinline__ uint32_t pack4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    return __byte_perm(__byte_perm(a, b, 0x0040), __byte_perm(c, d, 0x0040), 0x5410);
}

// A ring stage may only be refilled once the bytes read from it sit in registers: a shared-memory
// load is complete when its destination register is written, and neither `mbarrier` operations nor
// a TMA issue wait for loads in flight (round 1, DESIGN "hardware findings" 2: with the LSU queue
// backed up by slow peer/host stores an LDS waited long enough for the next TMA to overwrite the
// stage under it).  So the values loaded from the stage are folded, through a kernel parameter that
// is always zero but unknown to the compiler, into the ADDRESS operand of the refilling TMA.  The
// warp is converged across the loads (they are unconditional), a warp-level load completes as a
// whole, so lane 0's registers stand for all lanes.
__device__ __forceinline__ uint32_t stage_dep(const uint32_t (&w)[8], uint32_t zero) {
    return (w[0] | w[1] | w[2] | w[3] | w[4] | w[5] | w[6] | w[7]) & zero;
}

// One TMA descriptor per box shape of the plan, passed in the kernel's parameter block
// (__grid_constant__): descriptors in param space need no tensormap-proxy fence, unlike a table in
// global memory written by cudaMemcpy (a per-unit fence there drains every outstanding load of the
// warp and invalidates the SM's descriptor cache).
struct RingTmaps {
    CUtensorMap m[kMaxShapes];
};

struct RingUnit {     // what the warp knows about one of its upcoming units (all warp-uniform)
    uint32_t ticket;  // unit index; >= nunits: none
    uint32_t tile, f0, nf;
    uint32_t dy, dz, dw;  // words 1..3 of the tile's descriptor: box origin | plate, type, box shape | screen origin
};
__device__ __forceinline__ uint32_t unit_type(const RingUnit &u) { return (u.dz >> 8) & kTileTypeMask; }

// eight 32-bit streaming stores in ONE asm statement: all eight addresses are live at once, so the
// stores issue back to back (with one store per statement the compiler recycled a single address
// register pair and every store waited for the previous one to read its operands)
__device__ __forceinline__ void st_stream_u32x8(const uint64_t (&a)[8], const uint32_t (&w)[8]) {
    asm volatile(
        "st.global.cs.u32 [%0], %8;\n\t"
        "st.global.cs.u32 [%1], %9;\n\t"
        "st.global.cs.u32 [%2], %10;\n\t"
        "st.global.cs.u32 [%3], %11;\n\t"
        "st.global.cs.u32 [%4], %12;\n\t"
        "st.global.cs.u32 [%5], %13;\n\t"
        "st.global.cs.u32 [%6], %14;\n\t"
        "st.global.cs.u32 [%7], %15;"
        ::"l"(a[0]), "l"(a[1]), "l"(a[2]), "l"(a[3]), "l"(a[4]), "l"(a[5]), "l"(a[6]), "l"(a[7]),
          "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]), "r"(w[4]), "r"(w[5]), "r"(w[6]), "r"(w[7])
        : "memory");
}

// ---- gather role of the ring kernel's launch ---------------------------------------------------------------
// GATHER tiles (plate seams, singular points, boxes too large to stage) read the globe directly: 32-bit
// entries, lane = column, so one warp-level load covers 32 consecutive screen pixels of one row.  They are
// bound by load latency, so they get plain parallelism: one extra one-warp CTA per (tile, 8 of its rows, 4
// frames) behind the ring CTAs in the same grid.  The launch leaves shared memory for two of them per SM next
// to the resident ring warps, so this work runs beside the ring warps from the start and fills the slots they
// vacate at the end.  (kGatherRows, kGatherFrames: launch_plan.h)

template <bool RUBIX, bool RGBA, bool KEEP, bool TABLES, bool LAYOUT>
__device__ __forceinline__ void gather_item(const RingParams &p, uint32_t item, uint32_t lane, const FaceLayoutParams &lay) {
    const uint32_t nfg = (p.nframes + kGatherFrames - 1) / kGatherFrames;
    const uint32_t fg = item % nfg, rest = item / nfg;
    const uint32_t rg = rest % (kTileH / kGatherRows), gt = rest / (kTileH / kGatherRows);
    const uint4 d = __ldg(reinterpret_cast<const uint4 *>(p.tiles + p.nbox + gt));
    const uint32_t tile_x = d.w & 0xffffu, tile_y = (d.w >> 16) + rg * kGatherRows;
    const uint32_t width = static_cast<uint32_t>(p.width), height = static_cast<uint32_t>(p.height);
    const uint32_t f0 = fg * kGatherFrames, f1 = min(f0 + kGatherFrames, p.nframes);
    const uint32_t x = tile_x + lane;
    const uint32_t *__restrict__ ent32 = reinterpret_cast<const uint32_t *>(p.entries + d.x) + rg * kGatherRows * kTileW;
    uint32_t e[kGatherRows];
#pragma unroll
    for (int j = 0; j < kGatherRows; ++j) e[j] = __ldg(ent32 + j * kTileW + lane);
    if (x >= width) return;
    size_t at[kGatherRows];   // LAYOUT: the entries' byte offsets in a frame, split once for all frames
    if (LAYOUT) {
#pragma unroll
        for (int j = 0; j < kGatherRows; ++j) at[j] = layout_texel(e[j] & BLINKY_LM_INDEX_MASK, lay);
    }
    uint32_t v[kGatherFrames][kGatherRows];
#pragma unroll
    for (int g = 0; g < kGatherFrames; ++g) {
        const uint32_t f = f0 + g;
        const uint8_t *__restrict__ faces = p.faces + static_cast<size_t>(f < f1 ? f : f0) * p.face_stride;
#pragma unroll
        for (int j = 0; j < kGatherRows; ++j) {
            v[g][j] = 0x100u;   // "take the background"
            if (e[j] & BLINKY_LM_VALID) v[g][j] = ld_face(LAYOUT ? faces + at[j] : faces + (e[j] & BLINKY_LM_INDEX_MASK));
        }
    }
#pragma unroll
    for (int j = 0; j < kGatherRows; ++j) {
        const uint32_t y = tile_y + j;
        if (y >= height) break;
        if (KEEP && !(e[j] & BLINKY_LM_VALID)) continue;
        const size_t pix = static_cast<size_t>(y) * width + x;         // background index
        const size_t opix = static_cast<size_t>(y) * p.out_pitch + x;  // output index
        uint32_t bgv = 0, t = BLINKY_LM_TINT_NONE;
        if (!(e[j] & BLINKY_LM_VALID)) bgv = __ldg(p.bg + pix);
        else if (RUBIX) t = (e[j] >> BLINKY_LM_TINT_SHIFT) & 7u;
#pragma unroll
        for (int g = 0; g < kGatherFrames; ++g) {
            if (f0 + g >= f1) break;
            uint32_t b = v[g][j] & 0x100u ? bgv : v[g][j];
            if (RUBIX && t != BLINKY_LM_TINT_NONE) b = __ldg(p.lut + t * 256 + b);
            uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(f0 + g) * p.out_stride;
            const uint32_t *table = TABLES ? p.rgba + static_cast<size_t>(f0 + g) * p.table_words : p.rgba;
            if (RGBA) reinterpret_cast<uint32_t *>(o)[opix] = __ldg(table + b);
            else o[opix] = static_cast<uint8_t>(b);
        }
    }
}

// A dynamic ticket has been drawn: `d` is the counter value the warp received (warp-uniform).  Draws on one address
// are totally ordered and a launch makes exactly p.ndraws of them from 0, so the warp that receives ndraws - 1 makes
// the launch's last draw, and it stores 0: the next launch on the counter (stream order, or the next replay of a
// graph) starts from 0 without the host knowing what the counter holds.  Returns the unit index.
__device__ __forceinline__ uint32_t ticket_drawn(const RingParams &p, uint32_t d, uint32_t nw, uint32_t lane) {
    if (d == p.ndraws - 1u && lane == 0) asm volatile("st.relaxed.gpu.global.u32 [%0], 0;" ::"l"(p.ticket) : "memory");
    return p.nstatic * nw + d;
}

// CTAs per SM the ring kernel's register allocation is sized for, ring warps plus the gather CTAs beside them:
// 128 registers per thread (the BOX path uses 96, 116 with the rubix overlay).  How many ring warps are resident is
// decided in launch_ring.
constexpr int kRingMinBlocks = 16;

// KEEP (keep_unmapped): only mapped pixels are written.  The host gives this instance the BOX tiles alone (EMPTY tiles
// have nothing to write); a partly mapped quad is stored pixel by pixel and the background is never read.
// LAYOUT: the tensor maps view each frame's surface, (x, y, 1, frame); a unit's box origin is moved from plate to
// surface coordinates by the plate's origin when the issue cursor enters the unit.  Boxes that overhang their plate
// stage neighbouring texels, which no entry refers to.
template <bool RUBIX, bool RGBA, bool KEEP, bool TABLES, bool LAYOUT>
__global__ void __launch_bounds__(32, kRingMinBlocks) warp_ring_kernel(const __grid_constant__ RingParams p, const __grid_constant__ RingTmaps tm,
                                                                      const __grid_constant__ FaceLayoutParams lay) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // XOR with a parameter that is always zero: keeps ptxas from re-reading the special register
    // (S2R, tens of cycles) at every `lane == 0` test instead of holding the lane number in a register
    const uint32_t lane = threadIdx.x ^ p.zero;
    if (blockIdx.x >= p.ring_grid) {   // the CTAs behind the ring warps: one gather item each
        gather_item<RUBIX, RGBA, KEEP, TABLES, LAYOUT>(p, blockIdx.x - p.ring_grid, lane, lay);
        return;
    }
    const uint32_t R = p.ring_bytes;
    const uint32_t ring = smem_u32(smem_raw);
    uint8_t *tail = smem_raw + static_cast<size_t>(R);
    const uint32_t bars = smem_u32(tail);                             // kRingBoxes barriers, one per item in flight
    uint8_t *s_lut = tail + kRingBarBytes;                            // [6][256] plate LUTs
    uint32_t *s_rgba = reinterpret_cast<uint32_t *>(s_lut + (RUBIX ? 6 * 256 : 0));
    if (lane == 0) {
        for (uint32_t s = 0; s < kRingBoxes; ++s) mbar_init(bars + 8 * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (RUBIX) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.lut);
        uint32_t *dst = reinterpret_cast<uint32_t *>(s_lut);
        for (uint32_t i = lane; i < 6 * 256 / 4; i += 32) dst[i] = __ldg(src + i);
    }
    if (RGBA && !TABLES) {
        for (uint32_t i = lane; i < 256; i += 32) s_rgba[i] = __ldg(p.rgba + i);
    }
    __syncwarp();
    const uint32_t lut_base = smem_u32(s_lut);

    // TABLES: s_rgba holds one frame's table at a time, restaged before the first lookup of a frame whose table it
    // does not hold.  Each lane keeps its 8 words of the table it will need next in registers (two 128-bit loads,
    // issued a frame ahead), so the load latency hides behind a frame of work.  These are plain loads and stores of
    // this warp alone: __syncwarp orders the lookups in the old table before the stores of the new one, and those
    // before the next lookups.  The hazard stage_dep guards against (a TMA write overtaking a shared load still in
    // flight) does not arise: nothing in the async proxy writes s_rgba.
    uint32_t tab_f = 0xffffffffu, next_f = 0xffffffffu;   // frame whose table s_rgba holds / the registers hold
    uint4 next_t0 = make_uint4(0u, 0u, 0u, 0u), next_t1 = next_t0;
    auto fetch_table = [&](uint32_t f) {
        const uint4 *src = reinterpret_cast<const uint4 *>(p.rgba + static_cast<size_t>(f) * p.table_words) + 2 * lane;
        next_t0 = __ldg(src);
        next_t1 = __ldg(src + 1);
        next_f = f;
    };
    // s_rgba := frame f's table; then the registers start loading frame `after`'s
    auto use_table = [&](uint32_t f, uint32_t after) {
        if (tab_f != f) {
            if (next_f != f) fetch_table(f);
            __syncwarp();
            uint4 *dst = reinterpret_cast<uint4 *>(s_rgba) + 2 * lane;
            dst[0] = next_t0;
            dst[1] = next_t1;
            __syncwarp();
            tab_f = f;
        }
        if (after != tab_f && after != next_f) fetch_table(after);
    };

    const uint32_t NW = p.ring_grid;
    const uint32_t width = static_cast<uint32_t>(p.width), height = static_cast<uint32_t>(p.height);

    auto describe = [&](uint32_t ticket) {
        RingUnit u;
        u.ticket = ticket;
        u.tile = 0; u.f0 = 0; u.nf = 0; u.dy = 0; u.dz = 0; u.dw = 0;
        if (ticket < p.nunits) {
            u.tile = ticket / p.nchunks;
            const uint32_t chunk = ticket - u.tile * p.nchunks;
            u.f0 = chunk * p.fchunk;
            u.nf = min(p.fchunk, p.nframes - u.f0);
            // the ring kernel's tiles: the plan's BOX tiles [0, nbox), then its EMPTY tiles (the GATHER tiles in between
            // belong to the gather kernel)
            const uint4 d = __ldg(reinterpret_cast<const uint4 *>(p.tiles + (u.tile < p.nbox ? u.tile : u.tile + p.ngather)));
            u.dy = d.y; u.dz = d.z; u.dw = d.w;
        }
        return u;
    };
    auto is_box = [&](const RingUnit &u) { return u.ticket < p.nunits && u.tile < p.nbox; };
    // Work distribution: the first `nstatic` units of a warp are fixed (w, w + NW, ...), the rest of the
    // launch is handed out through the ticket counter.  Mostly static because one counter serves the
    // whole GPU and same-address atomics serialise; the dynamic tail evens out the finish.
    // A warp draws only while its last known ticket was good, so that the number of draws per launch is
    // a function of the launch alone (the host passes it as ndraws).
    uint32_t k_next = 0;        // index of the next ticket of this warp
    bool last_good = true;
    auto draw_now = [&]() {     // the k_next-th ticket, waiting for the counter if it is a dynamic one
        uint32_t t = 0xffffffffu;
        if (k_next < p.nstatic) {
            t = blockIdx.x + k_next * NW;
        } else if (last_good) {
            uint32_t d = 0;
            if (lane == 0) asm volatile("atom.global.add.u32 %0, [%1], 1;" : "=r"(d) : "l"(p.ticket) : "memory");
            t = ticket_drawn(p, __shfl_sync(0xffffffffu, d, 0), NW, lane);
        }
        ++k_next;
        last_good = t < p.nunits;
        return t;
    };
    RingUnit A = describe(draw_now());
    RingUnit B = describe(draw_now());
    RingUnit C = describe(draw_now());

    // Ring state (warp-uniform).  The ring is a byte FIFO of ITEMS — per BOX unit its entry block (bulk copy) followed by
    // one box per frame (TMA tensor load): an item goes behind the previous one, or at offset 0 when it would run over
    // the end — a rule the consuming side repeats with the same sizes, so no positions are passed along.  Small boxes
    // cost small space; the entry block of the next unit(s) is on its way while this unit's frames are warped, as deep
    // as the cursor may run ahead (single-frame launches: entry blocks and boxes of two units on).
    //   ipos   where the next box goes        cpos   end of the last consumed box (everything in flight lies
    //   is/cs  barrier slot of the next box to issue / to consume, phases: their parity bits     behind it)
    uint32_t cs = 0, is = 0, phases = 0, inflight = 0, ipos = 0, cpos = 0;
    auto room_for = [&](uint32_t n) {   // can a box of n bytes be placed now?
        if (inflight == 0) return true;                     // (n <= R: the planner caps boxes at the ring size)
        if (ipos > cpos) return ipos + n <= R || n <= cpos; // in flight: [cpos, ipos)
        return ipos + n <= cpos;                            // in flight: [cpos, R) and [0, ipos)
    };
    // Issue cursor: the next item of the warp's sequence — this unit's entry block and frames in order, then those of
    // the next BOX units (single-frame launches, the in-engine shape, need the look-ahead to reach two units on).
    // Its TMA operands are worked out when the cursor enters a unit, not per item.
    //   c_unit   0/1/2 = A/B/C: the unit the cursor is in (c_left > 0) or will look at next (c_left == 0)
    //   c_left   items of that unit still to issue (entry block + frames), c_entry: the next one is the entry block
    uint32_t c_unit = 0, c_left = 0, c_frame = 0, c_bytes = 0, c_tile = 0;
    bool c_entry = false;
    uint64_t c_tmap = 0;
    int c_bx = 0, c_by = 0, c_plate = 0;
    auto seat = [&]() {   // move the cursor to the first unit at or after c_unit that still has boxes to issue
        while (c_left == 0 && c_unit < 3) {
            // (field-wise selects: a reference chosen at run time would put the units on the stack)
            const uint32_t ticket = c_unit == 0 ? A.ticket : c_unit == 1 ? B.ticket : C.ticket;
            const uint32_t tile = c_unit == 0 ? A.tile : c_unit == 1 ? B.tile : C.tile;
            if (ticket < p.nunits && tile < p.nbox) {
                const uint32_t dy = c_unit == 0 ? A.dy : c_unit == 1 ? B.dy : C.dy;
                const uint32_t dz = c_unit == 0 ? A.dz : c_unit == 1 ? B.dz : C.dz;
                c_left = (c_unit == 0 ? A.nf : c_unit == 1 ? B.nf : C.nf) + 1u;
                c_entry = true;
                c_tile = tile;
                c_frame = c_unit == 0 ? A.f0 : c_unit == 1 ? B.f0 : C.f0;
                c_tmap = reinterpret_cast<uint64_t>(&tm.m[(dz >> (8 + kTileShapeShift)) & 63u]);
                c_bx = static_cast<int16_t>(dy & 0xffffu);
                c_by = static_cast<int16_t>(dy >> 16);
                c_plate = static_cast<int>(dz & 7u);
                if (LAYOUT) {
                    c_bx += lay.org_x[c_plate];
                    c_by += lay.org_y[c_plate];
                    c_plate = 0;
                }
                c_bytes = ((dz >> 16) & 0xffu) * (dz >> 24) * 128u;
            } else {
                ++c_unit;  // GATHER / EMPTY / no unit: nothing to stage
            }
        }
    };
    auto can_issue = [&]() { return c_left > 0 && inflight < p.max_inflight && room_for(c_entry ? static_cast<uint32_t>(kBoxBlockBytes) : c_bytes); };
    auto issue = [&](uint32_t dep) {   // precondition: can_issue()
        const uint32_t n = c_entry ? static_cast<uint32_t>(kBoxBlockBytes) : c_bytes;
        if (inflight == 0) ipos = cpos = 0;   // (an empty ring restarts at the front: keeps "everything in flight lies behind cpos" true)
        if (ipos + n > R) ipos = 0;
        if (lane == 0) {
            const uint32_t bar = bars + 8 * is;
            mbar_expect_tx(bar, n);
            if (c_entry) bulk_load(ring + ipos + dep, p.entries + static_cast<size_t>(c_tile) * kBoxBlockBytes, n, bar);
            else tma_load_box(ring + ipos + dep, reinterpret_cast<const CUtensorMap *>(c_tmap), c_bx, c_by, c_plate, static_cast<int>(c_frame), bar);
        }
        ipos += n;
        is = is + 1 == kRingBoxes ? 0 : is + 1;
        ++inflight;
        if (c_entry) c_entry = false;
        else ++c_frame;
        if (--c_left == 0) {
            ++c_unit;
            seat();
        }
    };

    while (A.ticket < p.nunits) {
        // look ahead: next ticket, B's entries.  asm volatile keeps a dynamic draw HERE, a whole unit
        // before its result is needed.
        const bool draw_dynamic = k_next >= p.nstatic && last_good;
        uint32_t drawn = 0;
        if (draw_dynamic && lane == 0) asm volatile("atom.global.add.u32 %0, [%1], 1;" : "=r"(drawn) : "l"(p.ticket) : "memory");

        const uint32_t tile_x = A.dw & 0xffffu, tile_y = A.dw >> 16;
        const uint32_t type = unit_type(A);
        seat();
        if (A.tile < p.nbox) {
            while (can_issue()) issue(0);
            const uint32_t a_bytes = ((A.dz >> 16) & 0xffu) * (A.dz >> 24) * 128u;   // size of this unit's boxes
            // ---- the lane's 32 entries, out of the ring into registers once for all frames of the unit
            mbar_wait(bars + 8 * cs, (phases >> cs) & 1u);
            if (cpos + kBoxBlockBytes > R) cpos = 0;
            const uint32_t ebuf = ring + cpos;
            uint4 eA[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) eA[k] = lds_v4(ebuf + (k * 32 + lane) * 16);
            uint32_t tintedA = 0;
            if (RUBIX) tintedA = lds_u32(ebuf + kBoxEntryBytes + lane * 4);
            phases ^= 1u << cs;
            cs = cs + 1 == kRingBoxes ? 0 : cs + 1;
            cpos += kBoxBlockBytes;
            --inflight;
            uint32_t off[32];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t w4[4] = {eA[k].x, eA[k].y, eA[k].z, eA[k].w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    off[8 * k + 2 * j] = w4[j] & kBoxOffsetMask;
                    off[8 * k + 2 * j + 1] = (w4[j] >> 16) & kBoxOffsetMask;
                }
            }
            // the block's bytes may be overwritten once they sit in registers (same reasoning as stage_dep)
            {
                uint32_t dep = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) dep |= eA[k].x | eA[k].y | eA[k].z | eA[k].w;
                dep = (dep | tintedA) & p.zero;
                while (can_issue()) issue(dep);
            }
            // rubix overlay: one LUT row for the tile, a byte mask per quad of the pixels it applies to
            uint32_t tmask[8];
            const uint32_t tile_tint = (A.dz >> 3) & 7u;
            const bool tinted_tile = RUBIX && tile_tint != kTileTintNone;
            const uint32_t lut_row = lut_base + (tile_tint & 7u) * 256u;
            if (RUBIX) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const uint32_t n = (tintedA >> (4 * q)) & 15u;
                    // bits 0..3 -> bytes 0..3 set to 0xff
                    tmask[q] = ((n & 1u) | ((n & 2u) << 7) | ((n & 4u) << 14) | ((n & 8u) << 21)) * 255u;
                }
            }
            // pixels of quad q (0..7): row (lane>>3) + 4q, columns 4*(lane&7) .. +3
            const uint32_t qx = tile_x + 4u * (lane & 7u), qy = tile_y + (lane >> 3);
            const size_t opx = RGBA ? 4 : 1;
            uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(A.f0) * p.out_stride + (static_cast<size_t>(qy) * p.out_pitch + qx) * opx;
            const uint32_t row4 = p.out_pitch * 4u * static_cast<uint32_t>(opx);   // four screen rows, bytes

            // one frame: wait for its box, 32 byte loads from shared memory, pack, hand the stage on
            auto gather_frame = [&](uint32_t (&w)[8]) {
                mbar_wait(bars + 8 * cs, (phases >> cs) & 1u);
                if (cpos + a_bytes > R) cpos = 0;
                const uint32_t base = ring + cpos;
                uint32_t b[32];
#pragma unroll
                for (int i = 0; i < 32; ++i) b[i] = lds_u8(base + off[i]);
#pragma unroll
                for (int q = 0; q < 8; ++q) w[q] = pack4(b[4 * q], b[4 * q + 1], b[4 * q + 2], b[4 * q + 3]);
                phases ^= 1u << cs;
                cs = cs + 1 == kRingBoxes ? 0 : cs + 1;
                cpos += a_bytes;
                --inflight;
                const uint32_t dep = stage_dep(w, p.zero);
                if (tinted_tile) {
                    // the tile's LUT row applied to every pixel, merged where the pixel is tinted
#pragma unroll
                    for (int i = 0; i < 32; ++i) b[i] = lds_u8(lut_row + b[i]);
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        const uint32_t t = pack4(b[4 * q], b[4 * q + 1], b[4 * q + 2], b[4 * q + 3]);
                        w[q] = (t & tmask[q]) | (w[q] & ~tmask[q]);
                    }
                }
                while (can_issue()) issue(dep);
            };
            auto store_rgba = [&](uint8_t *dst, uint32_t v) {
                st_stream_v4(reinterpret_cast<uint4 *>(dst), make_uint4(s_rgba[v & 0xffu], s_rgba[(v >> 8) & 0xffu], s_rgba[(v >> 16) & 0xffu], s_rgba[v >> 24]));
            };

            // (TABLES: the next frame is this unit's next, or the first of the unit after it)
            auto next_frame = [&](uint32_t f) { return f + 1 < A.nf ? A.f0 + f + 1 : B.f0; };

            if (type == TILE_BOX_FULL) {
                for (uint32_t f = 0; f < A.nf; ++f) {
                    uint32_t w[8];
                    gather_frame(w);
                    if (TABLES) use_table(A.f0 + f, next_frame(f));
                    if (RGBA) {
#pragma unroll
                        for (int q = 0; q < 8; ++q) store_rgba(o + static_cast<size_t>(static_cast<uint32_t>(q) * row4), w[q]);
                    } else {
                        uint64_t a[8];
#pragma unroll
                        for (int q = 0; q < 8; ++q) a[q] = reinterpret_cast<uint64_t>(o) + static_cast<uint64_t>(static_cast<uint32_t>(q) * row4);
                        st_stream_u32x8(a, w);
                    }
                    o += p.out_stride;
                }
            } else {
                // partly mapped tile, or one that hangs over the frame edge: per quad a byte mask of the
                // mapped pixels, the background word for the others, and whether the quad is stored at all
                uint32_t vmask[8], bgw[8];
                uint32_t store_mask = 0;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const uint32_t w0 = q & 1 ? eA[q >> 1].z : eA[q >> 1].x, w1 = q & 1 ? eA[q >> 1].w : eA[q >> 1].y;
                    uint32_t m = 0;  // valid bits (bit 15 of each 16-bit entry) -> byte masks
                    if (w0 & 0x8000u) m |= 0x000000ffu;
                    if (w0 & 0x80000000u) m |= 0x0000ff00u;
                    if (w1 & 0x8000u) m |= 0x00ff0000u;
                    if (w1 & 0x80000000u) m |= 0xff000000u;
                    vmask[q] = m;
                    const uint32_t y = qy + 4u * q;
                    bgw[q] = 0;
                    if (qx < width && y < height && (!KEEP || m != 0)) {   // (KEEP: an unmapped quad is skipped)
                        store_mask |= 1u << q;
                        if (!KEEP && m != 0xffffffffu) bgw[q] = __ldg(reinterpret_cast<const uint32_t *>(p.bg + static_cast<size_t>(y) * width + qx)) & ~m;
                    }
                }
                for (uint32_t f = 0; f < A.nf; ++f) {
                    uint32_t w[8];
                    gather_frame(w);
                    if (TABLES) use_table(A.f0 + f, next_frame(f));
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        if (!((store_mask >> q) & 1u)) continue;
                        uint8_t *dst = o + static_cast<size_t>(static_cast<uint32_t>(q) * row4);
                        if (KEEP && vmask[q] != 0xffffffffu) {
                            // partly mapped quad: its mapped pixels one by one
                            uint32_t px[4];
#pragma unroll
                            for (int k = 0; k < 4; ++k) px[k] = RGBA ? s_rgba[(w[q] >> (8 * k)) & 0xffu] : (w[q] >> (8 * k)) & 0xffu;
                            const uint32_t m = vmask[q];
                            st_quad_masked<RGBA>(dst, px, (m & 1u) | ((m >> 7) & 2u) | ((m >> 14) & 4u) | ((m >> 21) & 8u));
                            continue;
                        }
                        const uint32_t v = (w[q] & vmask[q]) | bgw[q];
                        if (RGBA) store_rgba(dst, v);
                        else st_stream_u32(reinterpret_cast<uint32_t *>(dst), v);
                    }
                    o += p.out_stride;
                }
            }
        } else if (!KEEP) {
            // ---- EMPTY: background only (quad layout)
            const uint32_t qx = tile_x + 4u * (lane & 7u), qy = tile_y + (lane >> 3);
            if (qx < width) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const uint32_t y = qy + 4u * q;
                    if (y >= height) break;
                    const size_t pix = static_cast<size_t>(y) * width + qx;
                    const uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(p.bg + pix));
                    const size_t opix = static_cast<size_t>(y) * p.out_pitch + qx;
                    for (uint32_t f = 0; f < A.nf; ++f) {
                        uint8_t *out_frame = static_cast<uint8_t *>(p.out) + static_cast<size_t>(A.f0 + f) * p.out_stride;
                        if (TABLES) {   // (s_rgba may hold another frame's table: looked up like K3)
                            const uint32_t *t = p.rgba + static_cast<size_t>(A.f0 + f) * p.table_words;
                            st_stream_v4(reinterpret_cast<uint4 *>(out_frame) + (opix >> 2),
                                         make_uint4(__ldg(t + (v & 0xffu)), __ldg(t + ((v >> 8) & 0xffu)), __ldg(t + ((v >> 16) & 0xffu)), __ldg(t + (v >> 24))));
                        } else if (RGBA) st_stream_v4(reinterpret_cast<uint4 *>(out_frame) + (opix >> 2),
                                                      make_uint4(s_rgba[v & 0xffu], s_rgba[(v >> 8) & 0xffu], s_rgba[(v >> 16) & 0xffu], s_rgba[v >> 24]));
                        else st_stream_u32(reinterpret_cast<uint32_t *>(out_frame) + (opix >> 2), v);
                    }
                }
            }
        }
        // rotate: A <- B <- C <- the ticket drawn above; the cursor moves with its unit
        uint32_t next_ticket = 0xffffffffu;
        if (k_next < p.nstatic) next_ticket = blockIdx.x + k_next * NW;
        else if (draw_dynamic) next_ticket = ticket_drawn(p, __shfl_sync(0xffffffffu, drawn, 0), NW, lane);
        ++k_next;
        last_good = next_ticket < p.nunits;
        A = B;
        B = C;
        C = describe(next_ticket);
        c_unit = c_unit > 0 ? c_unit - 1 : 0;
    }
}

// --------------------------------------------------------------------------
// K3: the GATHER tiles (plate seams, singular points; thousands of them with minifying lenses, where a tile's
// texels do not fit a box), launched in front of the ring kernel, one CTA column per GATHER tile (tiles
// [first_tile, first_tile + grid.x) of the plan); in short launches with few GATHER items they ride in the
// ring kernel's launch instead (gather_item, gather_rides_along).  Those tiles are bound
// by global-load latency and, at 32-byte sectors scattered over DRAM pages, by DRAM itself (ncu, 4K fisheye1:
// 4.6 TB/s = 70 % of the measured copy peak with about one useful byte in 20 fetched); they get plain parallelism: grid = (tiles, groups of 4 frames), 256 threads, a warp owns 4 tile rows and lane l is
// column l (one warp-level load = 32 consecutive screen pixels of one row).  The tile's entries are
// fetched once and reused for the frames of the group; all 16 gathers of a thread are issued before
// its first store.
// --------------------------------------------------------------------------
constexpr int kGatherFramesPerCta = 4;

template <bool RUBIX, bool RGBA, bool KEEP, bool TABLES, bool LAYOUT>
__global__ void __launch_bounds__(kThreads) warp_tile_gather_kernel(const __grid_constant__ RingParams p, const uint32_t first_tile,
                                                                    const __grid_constant__ FaceLayoutParams lay) {
    const uint32_t tid = threadIdx.x;
    const uint4 d = __ldg(reinterpret_cast<const uint4 *>(p.tiles + first_tile + blockIdx.x));
    const uint32_t type = (d.z >> 8) & kTileTypeMask;
    const uint32_t tile_x = d.w & 0xffffu, tile_y = d.w >> 16;
    const uint32_t width = static_cast<uint32_t>(p.width), height = static_cast<uint32_t>(p.height);
    const uint32_t f0 = blockIdx.y * kGatherFramesPerCta;
    const uint32_t f1 = min(f0 + kGatherFramesPerCta, p.nframes);

    // Never taken (the grid holds GATHER tiles only), but without it ptxas allocates the instances' registers differently
    // and the RGBA-with-layout one loses a CTA per SM: 8 % slower on the 16-frame 4K fisheye1 batch (H100, 700 W).
    if (type == TILE_EMPTY) {
        if (KEEP) return;   // nothing mapped, nothing to write
        // quad layout: thread t copies 4 background pixels of row t/8
        const uint32_t x = tile_x + (tid & 7u) * 4u, y = tile_y + (tid >> 3);
        if (x >= width || y >= height) return;
        const size_t pix = static_cast<size_t>(y) * width + x;
        const uint32_t bgw = __ldg(reinterpret_cast<const uint32_t *>(p.bg + pix));
        const uint32_t px[4] = {bgw & 0xffu, (bgw >> 8) & 0xffu, (bgw >> 16) & 0xffu, bgw >> 24};
        const size_t opix = static_cast<size_t>(y) * p.out_pitch + x;
        for (uint32_t f = f0; f < f1; ++f) {
            uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(f) * p.out_stride;
            const uint32_t *t = TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : p.rgba;
            if (RGBA) st_stream_v4(reinterpret_cast<uint4 *>(o) + (opix >> 2), make_uint4(__ldg(t + px[0]), __ldg(t + px[1]), __ldg(t + px[2]), __ldg(t + px[3])));
            else st_stream_u32(reinterpret_cast<uint32_t *>(o) + (opix >> 2), bgw);
        }
        return;
    }

    const uint32_t warp = tid >> 5, lane = tid & 31u;
    const uint32_t x = tile_x + lane;
    const uint32_t *__restrict__ ent32 = reinterpret_cast<const uint32_t *>(p.entries + d.x);
    uint32_t e[4], bgv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) e[j] = __ldg(ent32 + (warp * 4 + j) * kTileW + lane);
    if (x >= width) return;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t y = tile_y + warp * 4 + j;
        bgv[j] = 0;
        if (!KEEP && !(e[j] & BLINKY_LM_VALID) && y < height) bgv[j] = __ldg(p.bg + static_cast<size_t>(y) * width + x);
    }
    size_t at[4];   // LAYOUT: the entries' byte offsets in a frame, split once for all frames
    if (LAYOUT) {
#pragma unroll
        for (int j = 0; j < 4; ++j) at[j] = layout_texel(e[j] & BLINKY_LM_INDEX_MASK, lay);
    }
    uint32_t v[kGatherFramesPerCta][4];
#pragma unroll
    for (int g = 0; g < kGatherFramesPerCta; ++g) {
        const uint32_t f = f0 + g;
        const uint8_t *__restrict__ faces = p.faces + static_cast<size_t>(f < f1 ? f : f0) * p.face_stride;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            v[g][j] = bgv[j];
            if (e[j] & BLINKY_LM_VALID) v[g][j] = ld_face(LAYOUT ? faces + at[j] : faces + (e[j] & BLINKY_LM_INDEX_MASK));
        }
    }
#pragma unroll
    for (int g = 0; g < kGatherFramesPerCta; ++g) {
        const uint32_t f = f0 + g;
        if (f >= f1) break;
        uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(f) * p.out_stride;
        const uint32_t *table = TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : p.rgba;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t y = tile_y + warp * 4 + j;
            if (y < height && (!KEEP || (e[j] & BLINKY_LM_VALID))) {
                uint32_t b = v[g][j];
                if (RUBIX && (e[j] & BLINKY_LM_VALID)) {
                    const uint32_t t = (e[j] >> BLINKY_LM_TINT_SHIFT) & 7u;
                    if (t != BLINKY_LM_TINT_NONE) b = __ldg(p.lut + t * 256 + b);
                }
                const size_t pix = static_cast<size_t>(y) * p.out_pitch + x;
                if (RGBA) reinterpret_cast<uint32_t *>(o)[pix] = __ldg(table + b);
                else o[pix] = static_cast<uint8_t>(b);
            }
        }
    }
}

inline size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

// The flags of KernelVariant index I as constants: the kernels' template arguments.
template <int I>
struct VariantT {
    static constexpr bool rubix = I & 1, rgba = I & 2, keep = I & 4, tables = I & 8, layout = I & 16;
};

// Calls f(VariantT<v.index()>{}): the one place that turns the run-time flags into a kernel instance.  Only the
// indices that exist are instantiated.
template <int I = 0, typename F>
void with_variant(int index, F &&f) {
    if constexpr (I < 32) {
        if constexpr (KernelVariant::exists(I)) {
            if (index == I) return f(VariantT<I>{});
        }
        with_variant<I + 1>(index, f);
    }
}

constexpr uint32_t kCaptureSlots = 4096;   // work counters for captured ring launches (see WarpDevice::CaptureStream)

}  // namespace

int DeviceBuffer::alloc(size_t bytes) {
    reset();
    return cudaMalloc(&p_, bytes);
}

void DeviceBuffer::reset() {
    cudaFree(p_);
    p_ = nullptr;
}

// What one install makes resident: the lensmap's view, its map and tile plan, and the background.  Immutable once
// installed, except for the background's contents (set_background); captured graphs hold it (held_) while they may
// still read it.
struct WarpDevice::Generation {
    int width = 0, height = 0, platesize = 0, numplates = 0;
    size_t npix = 0, npix_pad = 0;
    int display[6] = {0, 0, 0, 0, 0, 0};
    int plate_rect[6][4] = {};
    std::vector<int32_t> span_off, spans;
    DeviceBuffer map;       // uint32_t[npix_pad]
    // tiled layout (ring kernel)
    bool have_plan = false, plan_has_box = false;
    DeviceBuffer tiles;     // TileDesc[ntiles]
    DeviceBuffer entries;   // entry_bytes of entry blocks
    size_t entry_bytes = 0;
    uint32_t ntiles = 0, nbox_tiles = 0, ngather_tiles = 0;
    int stage_bytes = 0;    // largest staged box of the plan
    std::vector<uint16_t> shapes;
    // uint8_t[npix_pad]: shared by the generations of one view size (see install)
    std::shared_ptr<DeviceBuffer> bg;
};

// ---------------------------------------------------------------------------
// frame pipeline slot: one frame of blinky_warp_host in flight
// ---------------------------------------------------------------------------
struct WarpDevice::Slot {
    ~Slot() {
        if (stream) cudaStreamDestroy(stream);
        if (done) cudaEventDestroy(done);
        if (h_faces) cudaFreeHost(h_faces);
        if (h_out) cudaFreeHost(h_out);
    }
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    DeviceBuffer d_faces, d_out;
    uint8_t *h_faces = nullptr, *h_out = nullptr;  // pinned staging
    bool busy = false;
    // finalize info
    uint8_t *dst = nullptr;          // the view origin of the caller's frame
    int dst_rowbytes = 0;
    bool keep_unmapped = false, direct = false;
};

struct WarpDevice::TmapSet {   // host-side: the descriptors travel in the kernel's parameter block
    const void *faces = nullptr;
    size_t face_stride = 0;
    int nframes = 0;
    uint32_t rowbytes = 0, rows = 0;   // face layout's surface (0: the dense [plate][ps][ps] frames)
    RingTmaps table;
    uint64_t last_use = 0;
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

#define CK(call)                                                  \
    do {                                                          \
        const cudaError_t e_ = static_cast<cudaError_t>(call);    \
        if (e_ != cudaSuccess) return fail(#call, e_);            \
    } while (0)

bool WarpDevice::fail(const char *what, int cuda_err) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(static_cast<cudaError_t>(cuda_err)));
    err_ = buf;
    return false;
}

WarpDevice::WarpDevice(int device) : device_(device) {
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaSetDevice: ") + cudaGetErrorString(e));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on sm_90 only
        char buf[256];
        snprintf(buf, sizeof buf, "blinky_b200 needs an sm_90 (H100) device; device %d is sm_%d%d (%s)", device, prop.major,
                 prop.minor, prop.name);
        throw std::runtime_error(buf);
    }
    sm_count_ = prop.multiProcessorCount;
    threads_per_sm_ = prop.maxThreadsPerMultiProcessor;
    smem_per_sm_ = prop.sharedMemPerMultiprocessor;
    if (const char *e = getenv("BLINKY_RING_BYTES")) ring_bytes_override_ = atoi(e);
    if (const char *e = getenv("BLINKY_RING_BOXES")) ring_boxes_ = atoi(e);
    if (const char *e = getenv("BLINKY_MERGED_ITEMS")) merged_items_max_ = atoi(e);
    if (const char *e = getenv("BLINKY_RING_CTAS")) ring_ctas_cap_ = atoi(e);
    if (const char *e = getenv("BLINKY_FCHUNK")) fchunk_ = atoi(e);
    if (const char *e = getenv("BLINKY_SERIAL_GATHER")) serial_gather_ = atoi(e) != 0;  // GATHER tiles in their own kernel before the ring kernel (A/B)
    if (const char *e = getenv("BLINKY_STATIC_PCT")) static_pct_ = std::max(0, std::min(100, atoi(e)));
    e = static_cast<cudaError_t>(d_lut_.alloc(6 * 256));
    if (e == cudaSuccess) e = cudaMemset(d_lut_.get(), 0, 6 * 256);
    if (e == cudaSuccess) e = static_cast<cudaError_t>(d_rgba_.alloc(256 * 4));
    if (e == cudaSuccess) e = cudaMemset(d_rgba_.get(), 0, 256 * 4);
    // (here, not on first use: a capture may allocate nothing)
    if (e == cudaSuccess) e = static_cast<cudaError_t>(d_capture_slots_.alloc(kCaptureSlots * sizeof(uint32_t)));
    if (e == cudaSuccess) e = cudaMemset(d_capture_slots_.get(), 0, kCaptureSlots * sizeof(uint32_t));
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaMalloc: ") + cudaGetErrorString(e));
}

// (the members then free what they own)
WarpDevice::~WarpDevice() {
    cudaSetDevice(device_);
    cudaDeviceSynchronize();
}

size_t WarpDevice::padded_pixels(size_t npix) { return round_up(npix, kPixelsPerBlock); }
int WarpDevice::width() const { return cur_ ? cur_->width : 0; }
int WarpDevice::height() const { return cur_ ? cur_->height : 0; }
int WarpDevice::platesize() const { return cur_ ? cur_->platesize : 0; }
size_t WarpDevice::plan_tiles() const { return cur_ && cur_->have_plan ? cur_->ntiles : 0; }
size_t WarpDevice::plan_entry_bytes() const { return cur_ && cur_->have_plan ? cur_->entry_bytes : 0; }

bool WarpDevice::download_lensmap(uint32_t *out) {
    CK(cudaSetDevice(device_));
    if (cur_) CK(cudaMemcpy(out, cur_->map.get(), cur_->npix * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return true;
}

bool WarpDevice::download_plan(void *tiles, void *entries, size_t entry_bytes) {
    CK(cudaSetDevice(device_));
    if (!plan_tiles()) return true;
    if (tiles) CK(cudaMemcpy(tiles, cur_->tiles.get(), cur_->ntiles * sizeof(TileDesc), cudaMemcpyDeviceToHost));
    if (entries && entry_bytes) CK(cudaMemcpy(entries, cur_->entries.get(), entry_bytes, cudaMemcpyDeviceToHost));
    return true;
}

bool WarpDevice::install(const LensmapUpload &lm, DevicePlan &&plan) {
    CK(cudaSetDevice(device_));
    CK(cudaDeviceSynchronize());  // nothing may still be reading the buffers freed or rewritten in place below
    auto g = std::make_shared<Generation>();
    g->width = lm.width;
    g->height = lm.height;
    g->platesize = lm.platesize;
    g->numplates = lm.numplates;
    g->npix = static_cast<size_t>(lm.width) * lm.height;
    g->npix_pad = padded_pixels(g->npix);
    memcpy(g->display, lm.display, sizeof g->display);
    memcpy(g->plate_rect, lm.plate_rect, sizeof g->plate_rect);
    g->span_off.assign(lm.span_off, lm.span_off + lm.height + 1);
    g->spans.assign(lm.spans, lm.spans + lm.nspans * 2);
    g->map = std::move(plan.d_map);
    if (plan.ntiles > 0) {
        g->tiles = std::move(plan.d_tiles);
        g->entries = std::move(plan.d_entries);
        g->ntiles = plan.ntiles;
        g->entry_bytes = plan.entry_bytes;
        g->nbox_tiles = static_cast<uint32_t>(plan.plan.n_box);
        g->ngather_tiles = static_cast<uint32_t>(plan.plan.n_gather);
        g->stage_bytes = plan.plan.stage_bytes;
        g->shapes = std::move(plan.plan.shapes);
        g->plan_has_box = plan.plan.n_box > 0;
        g->have_plan = true;
    }
    // The background stays shared, contents and all, while the view size stays the same.  A new view size starts from
    // zeros: in a new buffer when the padded size changes or a held generation (a captured graph) reads the old one,
    // otherwise in place.
    const Generation *old = cur_.get();
    if (old && old->width == g->width && old->height == g->height) {
        g->bg = old->bg;
    } else {
        bool reuse = old && old->npix_pad == g->npix_pad;
        for (const auto &h : held_) reuse = reuse && h->bg != old->bg;
        if (reuse) {
            g->bg = old->bg;
        } else {
            g->bg = std::make_shared<DeviceBuffer>();
            CK(g->bg->alloc(g->npix_pad));
        }
        CK(cudaMemset(g->bg->get(), 0, g->npix_pad));
    }
    if (!set_luts(lm.palmaps)) return false;
    rubix_ = lm.rubix;
    cur_ = std::move(g);   // (frees the old generation unless a captured graph holds it)
    tmap_sets_.clear();
    slots_.clear();        // frame slots depend on the sizes: rebuilt lazily
    return true;
}

bool WarpDevice::set_luts(const uint8_t palmaps[6 * 256]) {
    CK(cudaSetDevice(device_));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(d_lut_.get(), palmaps, 6 * 256, cudaMemcpyHostToDevice));
    return true;
}

bool WarpDevice::set_background(const uint8_t *bg_host) {
    if (!cur_) {
        err_ = "set_background: build a lensmap first (the background has the view's size)";
        return false;
    }
    CK(cudaSetDevice(device_));
    CK(cudaDeviceSynchronize());
    if (bg_host) CK(cudaMemcpy(cur_->bg->get(), bg_host, cur_->npix, cudaMemcpyHostToDevice));
    else CK(cudaMemset(cur_->bg->get(), 0, cur_->npix_pad));
    return true;
}

bool WarpDevice::set_rgba_table(const uint32_t table[256]) {
    CK(cudaSetDevice(device_));
    CK(cudaMemcpy(d_rgba_.get(), table, 256 * 4, cudaMemcpyHostToDevice));
    return true;
}

void WarpDevice::set_face_layout(int rowbytes, const int32_t *origins, int nplates) {
    layout_rowbytes_ = rowbytes > 0 ? rowbytes : 0;
    layout_origins_.assign(origins && rowbytes > 0 ? origins : nullptr, origins && rowbytes > 0 ? origins + 2 * nplates : nullptr);
}

WarpState WarpDevice::state(const GlobeState &globe) const {
    WarpState s;
    if (cur_) {
        s.width = cur_->width;
        s.height = cur_->height;
        s.platesize = cur_->platesize;
        s.display = cur_->display;
        s.plate_rect = cur_->plate_rect;
    }
    s.globe = globe;
    s.layout_rowbytes = layout_rowbytes_;
    s.layout_origins = layout_origins_.data();
    s.layout_plates = static_cast<int>(layout_origins_.size() / 2);
    return s;
}

bool WarpDevice::check(const WarpRequest &r, const RayRequest &q, const GlobeState &globe, CheckedWarp *c) {
    const int rc = check_warp(r, q, state(globe), c, &err_);
    err_code_ = rc != BLINKY_OK ? rc : BLINKY_E_CUDA;
    return rc == BLINKY_OK;
}

bool WarpDevice::capture_info(void *stream, bool *capturing, unsigned long long *id) {
    // (the legacy default stream cannot capture, and asking it while another stream captures is an error)
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    *id = 0;
    if (stream != nullptr && static_cast<cudaStream_t>(stream) != cudaStreamLegacy)
        CK(cudaStreamGetCaptureInfo(static_cast<cudaStream_t>(stream), &cap, id));
    *capturing = cap != cudaStreamCaptureStatusNone;
    return true;
}

void WarpDevice::remember_capture(void *stream, unsigned long long id) {
    if (held_.empty() || held_.back() != cur_) held_.push_back(cur_);
    bool known = false;
    for (CaptureStream &c : capture_streams_)
        if (c.stream == stream) c.id = id, known = true;
    if (!known) capture_streams_.push_back({stream, id});
}

bool WarpDevice::warp(const WarpRequest &r) {
    CheckedWarp c;
    if (!check(r, RayRequest(), GlobeState(), &c)) return false;
    if (!c.launch) return true;
    const Generation &g = *cur_;
    const KernelVariant v = {rubix_, r.rgba, r.keep_unmapped, r.rgba && r.tables && r.table_stride != 0, c.use_layout};
    const WarpKernel k = choose_kernel(r, c.pitch, c.use_layout ? &c.layout : nullptr, g.width, g.height, g.have_plan, g.plan_has_box,
                                       variant_ == BLINKY_KERNEL_GATHER);
    bool capturing = false;
    unsigned long long cap_id = 0;
    if (!capture_info(r.stream, &capturing, &cap_id)) return false;
    const bool ok = k == WarpKernel::Ring ? launch_ring(r, c, v, capturing) : launch_flat(r, c, v, k);
    if (capturing) remember_capture(r.stream, cap_id);
    return ok;
}

bool WarpDevice::warp_rays(const WarpRequest &r, const RayRequest &q, const GlobeState &globe, const LensBuildParams &params) {
    CheckedWarp c;
    if (!check(r, q, globe, &c)) return false;
    if (!c.launch) return true;
    const Generation &g = *cur_;
    bool capturing = false;
    unsigned long long cap_id = 0;
    if (!capture_info(r.stream, &capturing, &cap_id)) return false;
    const RayWarpLaunch L = {r,
                             q,
                             c,
                             g.bg->as<const uint8_t>(),
                             d_lut_.as<const uint8_t>(),
                             r.tables ? r.tables : d_rgba_.as<const uint32_t>(),
                             g.width,
                             g.height,
                             ray_warp_shape(r, q, c.pitch, g.width, g.height, static_cast<uint32_t>(sm_count_) * static_cast<uint32_t>(threads_per_sm_)),
                             rubix_,
                             params};
    int e = 0;
    const bool ok = launch_ray_warp(L, &last_kernel_, &e);
    launches_ += 1 + c.lmax;
    if (capturing) remember_capture(r.stream, cap_id);
    return ok ? true : fail(ray_warp_kernel_name(q.filter, q.factor), e);
}

bool WarpDevice::release_captures() {
    err_code_ = BLINKY_E_CUDA;
    // a capture that holds a warp of this object and is still open: synchronising now would invalidate it
    for (const CaptureStream &c : capture_streams_) {
        cudaStreamCaptureStatus s = cudaStreamCaptureStatusNone;
        unsigned long long id = 0;
        if (cudaStreamGetCaptureInfo(static_cast<cudaStream_t>(c.stream), &s, &id) == cudaSuccess && s != cudaStreamCaptureStatusNone &&
            id == c.id) {
            err_code_ = BLINKY_E_INVALID;
            err_ = "release_captures: a stream is still capturing a warp of this context (end the capture first)";
            return false;
        }
    }
    CK(cudaSetDevice(device_));
    const cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaErrorStreamCaptureUnsupported || e == cudaErrorStreamCaptureImplicit) {
        err_code_ = BLINKY_E_INVALID;
        return fail("release_captures: cudaDeviceSynchronize while a stream is capturing", e);
    }
    if (e != cudaSuccess) return fail("release_captures: cudaDeviceSynchronize", e);
    held_.clear();
    capture_streams_.clear();
    capture_slots_used_ = 0;
    return true;
}

WarpDevice::TmapSet *WarpDevice::get_tmaps(const void *d_faces, size_t face_stride, int nframes, uint32_t rowbytes, uint32_t rows) {
    const uint64_t tick = ++tmap_tick_;
    for (const auto &t : tmap_sets_)
        if (t->faces == d_faces && t->face_stride == face_stride && t->nframes == nframes && t->rowbytes == rowbytes && t->rows == rows) {
            t->last_use = tick;
            return t.get();
        }
    if (!encode_fn_) {
        cudaDriverEntryPointQueryResult qres;
        void *fn = nullptr;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
        if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
            fail("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled)", e);
            return nullptr;
        }
        encode_fn_ = fn;
    }
    TmapSet *t = nullptr;
    if (tmap_sets_.size() >= 32) {  // host memory only (a launch copies its table into the parameter block): recycle the oldest
        t = tmap_sets_[0].get();
        for (const auto &c : tmap_sets_)
            if (c->last_use < t->last_use) t = c.get();
    } else {
        tmap_sets_.push_back(std::make_unique<TmapSet>());
        t = tmap_sets_.back().get();
    }
    t->faces = d_faces;
    t->face_stride = face_stride;
    t->nframes = nframes;
    t->rowbytes = rowbytes;
    t->rows = rows;
    t->last_use = tick;
    memset(&t->table, 0, sizeof t->table);
    const Generation &g = *cur_;
    const cuuint64_t ps = static_cast<cuuint64_t>(g.platesize);
    // 4-D view of the globe: (x, y, plate, frame); with a face layout (rowbytes > 0) one frame's surface is the single
    // "plate": (x, y, 1, frame), rowbytes wide and `rows` high
    const cuuint64_t fw = rowbytes ? rowbytes : ps, fh = rowbytes ? rows : ps, np = rowbytes ? 1 : static_cast<cuuint64_t>(g.numplates);
    const cuuint64_t dims[4] = {fw, fh, np, static_cast<cuuint64_t>(nframes)};
    const cuuint64_t fstride = nframes > 1 ? static_cast<cuuint64_t>(face_stride) : fw * fh * np;
    const cuuint64_t strides[3] = {fw, fw * fh, fstride};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    for (size_t si = 0; si < g.shapes.size() && si < static_cast<size_t>(kMaxShapes); ++si) {
        const uint32_t w16 = g.shapes[si] >> 8, h8 = g.shapes[si] & 0xff;
        const cuuint32_t box[4] = {w16 * 16, h8 * 8, 1, 1};
        CUresult r = reinterpret_cast<EncodeTiledFn>(encode_fn_)(
            &t->table.m[si], CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void *>(d_faces), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            char buf[160];
            snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled(box %ux%u, ps %d) failed with CUresult %d", w16 * 16, h8 * 8, g.platesize, static_cast<int>(r));
            err_ = buf;
            t->faces = nullptr;
            return nullptr;
        }
    }
    return t;
}

// Resident ring warps per SM by default (BLINKY_RING_CTAS): measured on the 4K panini batch (bench.py, H100 80GB HBM3
// at a 400 W power limit) 8 / 10 / 12 / 14 / 16 warps give 578 / 578 / 657 / 652 / 653 Gpixel/s — beyond 12, more
// warps only spread the faces' L2 footprint; the registers left over go to the gather CTAs.
constexpr int kRingWarpsDefault = 12;

bool WarpDevice::launch_ring(const WarpRequest &r, const CheckedWarp &c, const KernelVariant &v, bool capturing) {
    cudaStream_t st = static_cast<cudaStream_t>(r.stream);
    const Generation &g = *cur_;
    RingParams p;
    p.tiles = g.tiles.as<const TileDesc>();
    p.entries = g.entries.as<const uint8_t>();
    static const RingTmaps kNoTmaps = {};
    const RingTmaps *tm = &kNoTmaps;
    if (g.plan_has_box) {
        TmapSet *t = get_tmaps(r.faces, r.face_stride, r.nframes, c.layout.rowbytes, v.layout ? c.layout_rows : 0u);
        if (!t) return false;
        tm = &t->table;
    }
    p.faces = static_cast<const uint8_t *>(r.faces);
    p.face_stride = r.face_stride;
    p.bg = g.bg->as<const uint8_t>();
    p.lut = d_lut_.as<const uint8_t>();
    p.rgba = r.tables ? r.tables : d_rgba_.as<const uint32_t>();
    p.table_words = static_cast<uint32_t>(r.table_stride / 4);
    p.out = c.view;
    p.out_stride = r.out_stride;
    p.out_pitch = static_cast<uint32_t>(c.pitch) / (v.rgba ? 4u : 1u);   // (whole pixels: an RGBA pitch is a multiple of 4 bytes)
    p.nbox = g.nbox_tiles;
    p.ngather = g.ngather_tiles;
    p.ntiles = g.ntiles;
    p.nframes = static_cast<uint32_t>(r.nframes);
    p.width = g.width;
    p.height = g.height;
    p.zero = 0;
    // The ring kernel's units are the BOX tiles [0, nbox) and the EMPTY tiles; with keep_unmapped an EMPTY tile has
    // nothing to write, and the units are the BOX tiles alone.  The GATHER tiles in between ride along as gather CTAs
    // or go to K3, launched in front on the same stream (gather_rides_along).
    const uint32_t nempty = g.ntiles - g.nbox_tiles - g.ngather_tiles;
    const uint32_t ring_tiles = g.nbox_tiles + (v.keep ? 0u : nempty);
    const size_t fixed = kRingBarBytes + (v.rubix ? 6 * 256 : 0) + (v.rgba ? 1024 : 0);
    const uint32_t max_box = std::max<uint32_t>(static_cast<uint32_t>(g.stage_bytes > 0 ? g.stage_bytes : 128), kBoxBlockBytes);  // largest ring item
    const bool merged_gather = gather_rides_along(g.ngather_tiles, r.nframes, merged_items_max_, serial_gather_);
    // as many ring warps per SM as the registers allow (or BLINKY_RING_CTAS), as far as shared memory lets them
    const RingGeometry geo = ring_geometry(smem_per_sm_, ring_ctas_cap_ > 0 ? std::min(ring_ctas_cap_, kRingMinBlocks) : kRingWarpsDefault,
                                           merged_gather, fixed, max_box, ring_bytes_override_);
    if (geo.warps < 1) {
        err_ = "ring kernel: the plan's largest box does not fit the staging ring";
        return false;
    }
    p.ring_bytes = geo.ring_bytes;
    // items in flight per warp: two boxes and (at unit boundaries) the next entry block (BLINKY_RING_BOXES overrides)
    p.max_inflight = static_cast<uint32_t>(std::max(1, std::min(ring_boxes_ > 0 ? ring_boxes_ : 3, kRingBoxes)));
    const size_t smem = static_cast<size_t>(geo.ring_bytes) + fixed;
    const int vi = v.index();
    if (ring_ctas_per_sm_[vi] == 0 || ring_smem_[vi] != smem) {
        int n = 0;
        cudaError_t e = cudaSuccess;
        with_variant(vi, [&](auto vt) {   // the instance's dynamic shared memory and occupancy
            using V = decltype(vt);
            auto *kernel = warp_ring_kernel<V::rubix, V::rgba, V::keep, V::tables, V::layout>;
            e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
            if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, 32, smem);
        });
        if (e != cudaSuccess) return fail("ring kernel configuration (shared memory / occupancy)", e);
        if (n < 1) {
            err_ = "ring kernel does not fit on an SM";
            return false;
        }
        ring_ctas_per_sm_[vi] = n;
        ring_smem_[vi] = smem;
    }
    int ctas = std::min(ring_ctas_per_sm_[vi], geo.warps);
    uint32_t grid = static_cast<uint32_t>(sm_count_ * ctas);
    const uint32_t fchunk = frames_per_unit(ring_tiles, p.nframes, grid, fchunk_);
    p.fchunk = fchunk;
    p.nchunks = (p.nframes + fchunk - 1) / fchunk;
    p.nunits = ring_tiles * p.nchunks;
    if (grid > p.nunits) grid = p.nunits;
    // The ring kernel's work counter, 0 before and after every launch (ticket_drawn).  Eager launches on one stream
    // run one after the other and share the stream's counter; a captured launch gets a pool slot of its own.  Taken
    // before anything is launched, so that a capture refused for want of slots launches nothing.
    if (grid > 0 && capturing) {
        if (capture_slots_used_ == kCaptureSlots) {
            err_code_ = BLINKY_E_STATE;
            err_ = "warp: all 4096 work counters for captured ring kernel launches are in use; call blinky_release_captures "
                   "once the graphs holding them will not run again";
            return false;
        }
        p.ticket = d_capture_slots_.as<uint32_t>() + capture_slots_used_++;
    } else if (grid > 0) {
        TicketCounter *tc = nullptr;
        for (TicketCounter &c : tickets_)
            if (c.stream == r.stream) tc = &c;
        if (!tc) {
            if (tickets_.size() >= 64) {  // streams come and go: start over
                CK(cudaDeviceSynchronize());
                tickets_.clear();
            }
            TicketCounter c;
            c.stream = r.stream;
            CK(c.counter.alloc(sizeof(uint32_t)));
            CK(cudaMemsetAsync(c.counter.get(), 0, sizeof(uint32_t), st));
            tickets_.push_back(std::move(c));
            tc = &tickets_.back();
        }
        p.ticket = tc->counter.as<uint32_t>();
    }
    char buf[640];
    int nbuf = 0;
    // GATHER tiles: K3 in front of the ring kernel, unless they ride in its launch (which needs ring units)
    snprintf(buf, sizeof buf, "%s", g.ngather_tiles == 0 && grid == 0 ? "no kernel: no tile of the view has a pixel to write" : "");
    if (g.ngather_tiles > 0 && (grid == 0 || !merged_gather)) {
        dim3 g2(g.ngather_tiles, static_cast<unsigned>((r.nframes + kGatherFramesPerCta - 1) / kGatherFramesPerCta));
        with_variant(vi, [&](auto vt) {
            using V = decltype(vt);
            warp_tile_gather_kernel<V::rubix, V::rgba, V::keep, V::tables, V::layout><<<g2, kThreads, 0, st>>>(p, g.nbox_tiles, c.layout);
        });
        ++launches_;
        snprintf(buf, sizeof buf, "warp_tile_gather_kernel<rubix=%d,rgba=%d%s> grid=(%u,%u) block=%d", v.rubix, v.rgba, v.tags(), g2.x, g2.y, kThreads);
    }
    if (grid > 0) {
        const TicketSchedule ts = ticket_schedule(p.nunits, grid, static_pct_);
        p.nstatic = ts.nstatic;
        p.ndraws = ts.ndraws;
        p.ring_grid = grid;
        const uint32_t extra = merged_gather ? gather_items(g.ngather_tiles, r.nframes) : 0u;
        with_variant(vi, [&](auto vt) {
            using V = decltype(vt);
            warp_ring_kernel<V::rubix, V::rgba, V::keep, V::tables, V::layout><<<grid + extra, 32, smem, st>>>(p, *tm, c.layout);
        });
        ++launches_;
        nbuf = static_cast<int>(strlen(buf));
        snprintf(buf + nbuf, sizeof buf - static_cast<size_t>(nbuf),
                 "%swarp_ring_kernel<rubix=%d,rgba=%d%s> grid=%u+%u block=32 (%d ring warps/SM, TMA box ring of %u B, <=%u boxes in flight, %u frames/unit, %u units; "
                 "%u gather CTAs of %dx32 px x %d frames)",
                 nbuf ? " + " : "", v.rubix, v.rgba, v.tags(), grid, extra, ctas, p.ring_bytes, p.max_inflight, fchunk, p.nunits, extra, kGatherRows,
                 kGatherFrames);
    }
    last_kernel_ = buf;
    CK(cudaGetLastError());
    return true;
}

bool WarpDevice::launch_flat(const WarpRequest &r, const CheckedWarp &c, const KernelVariant &v, WarpKernel k) {
    // NULL is CUDA's default stream (what torch.cuda.current_stream() hands out unless the caller made its own)
    cudaStream_t st = static_cast<cudaStream_t>(r.stream);
    const Generation &g = *cur_;
    WarpParams p;
    p.lensmap4 = g.map.as<const uint4>();
    p.faces = static_cast<const uint8_t *>(r.faces);
    p.face_stride = r.face_stride;
    p.bg32 = g.bg->as<const uint32_t>();
    p.lut = d_lut_.as<const uint8_t>();
    p.rgba = r.tables ? r.tables : d_rgba_.as<const uint32_t>();
    p.table_words = static_cast<uint32_t>(r.table_stride / 4);
    p.out = c.view;
    p.out_stride = r.out_stride;
    p.nquads = static_cast<uint32_t>((g.npix + 3) / 4);
    p.npix = static_cast<uint32_t>(g.npix);
    p.width = static_cast<uint32_t>(g.width);
    p.out_pitch = static_cast<uint32_t>(c.pitch);
    p.pitched = c.pitch != static_cast<size_t>(g.width) * (v.rgba ? 4 : 1);
    const bool vector = k == WarpKernel::Vector;
    const dim3 grid(static_cast<unsigned>(vector ? g.npix_pad / kPixelsPerBlock : (g.npix + kThreads - 1) / kThreads), static_cast<unsigned>(r.nframes));
    with_variant(v.index(), [&](auto vt) {
        using V = decltype(vt);
        if (vector) warp_gather_kernel<V::rubix, V::rgba, V::keep, V::tables, V::layout><<<grid, kThreads, 0, st>>>(p, c.layout);
        else warp_scalar_kernel<V::rubix, V::rgba, V::keep, V::tables, V::layout><<<grid, kThreads, 0, st>>>(p, c.layout);
    });
    char buf[160];
    snprintf(buf, sizeof buf, "%s<rubix=%d,rgba=%d%s> grid=(%u,%u) block=%d", vector ? "warp_gather_kernel" : "warp_scalar_kernel", v.rubix, v.rgba,
             v.tags(), grid.x, grid.y, kThreads);
    last_kernel_ = buf;
    ++launches_;
    CK(cudaGetLastError());
    return true;
}

bool WarpDevice::ensure_slots() {
    if (!slots_.empty()) return true;
    // three frames in flight overlap upload, warp and copy back; 2-8 measured the same
    constexpr int kSlots = 3;
    slot_face_bytes_ = static_cast<size_t>(cur_->numplates) * cur_->platesize * cur_->platesize;
    slot_out_bytes_ = round_up(cur_->npix, 16);
    for (int i = 0; i < kSlots; ++i) {
        slots_.push_back(std::make_unique<Slot>());
        Slot *s = slots_.back().get();
        CK(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&s->done, cudaEventDisableTiming));
        CK(s->d_faces.alloc(slot_face_bytes_));
        CK(cudaMemset(s->d_faces.get(), 0, slot_face_bytes_));
        CK(s->d_out.alloc(slot_out_bytes_));
        // (pinned staging for callers whose buffers are not pinned: allocated when first needed)
    }
    return true;
}

void WarpDevice::finalize_slot(Slot &s) {
    if (!s.busy) return;
    cudaEventSynchronize(s.done);
    s.busy = false;
    if (s.direct) return;  // the copy engine already wrote the caller's buffer
    const Generation &g = *cur_;
    const int W = g.width, H = g.height;
    uint8_t *dst = s.dst;
    if (s.keep_unmapped) {
        // only mapped pixels are written, like `if (*lmap)` in render_lensmap (:2413)
        for (int y = 0; y < H; ++y) {
            const uint8_t *src = s.h_out + static_cast<size_t>(y) * W;
            uint8_t *row = dst + static_cast<size_t>(y) * s.dst_rowbytes;
            for (int32_t j = g.span_off[static_cast<size_t>(y)]; j < g.span_off[static_cast<size_t>(y) + 1]; ++j) {
                const int32_t a = g.spans[static_cast<size_t>(j) * 2], b = g.spans[static_cast<size_t>(j) * 2 + 1];
                memcpy(row + a, src + a, static_cast<size_t>(b - a));
            }
        }
    } else if (s.dst_rowbytes == W) {
        memcpy(dst, s.h_out, static_cast<size_t>(W) * H);
    } else {
        for (int y = 0; y < H; ++y) memcpy(dst + static_cast<size_t>(y) * s.dst_rowbytes, s.h_out + static_cast<size_t>(y) * W, static_cast<size_t>(W));
    }
}

static bool is_pinned(const void *p) {
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();  // clear
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}

bool WarpDevice::warp_host(const WarpRequest &r) {
    CheckedWarp c;
    if (!check(r, RayRequest(), GlobeState(), &c)) return false;
    const Generation &g = *cur_;
    const uint8_t *faces_host = static_cast<const uint8_t *>(r.faces);
    const uint8_t *dst_host = static_cast<const uint8_t *>(r.out);
    const size_t face_stride = r.face_stride;
    const int dst_rowbytes = r.rowbytes, nframes = r.nframes;
    const bool keep_unmapped = r.keep_unmapped;
    // with a face layout the plates' rectangles are read out of each frame's surface; the device copy stays dense
    const FaceLayoutParams &lay = c.layout;
    const bool layout = c.use_layout;
    const size_t ps = static_cast<size_t>(g.platesize);
    const size_t src_pitch = layout ? lay.rowbytes : ps;
    CK(cudaSetDevice(device_));
    if (!ensure_slots()) return false;
    const size_t ps2 = ps * ps;
    // (one driver query per distinct buffer, not two per call)
    if (faces_host != pin_src_ptr_) pin_src_ptr_ = faces_host, pin_src_ = is_pinned(faces_host);
    if (dst_host != pin_dst_ptr_) pin_dst_ptr_ = dst_host, pin_dst_ = is_pinned(dst_host);
    const bool src_pinned = pin_src_, dst_pinned = pin_dst_;
    const int W = g.width, H = g.height;
    const bool direct = dst_pinned && !keep_unmapped;  // the copy engine writes the caller's buffer, no staging
    const size_t frame = static_cast<size_t>(W) * H;
    bool ok = true;
    int f = 0;
    for (; f < nframes; ++f) {
        Slot &s = *slots_[static_cast<size_t>(f) % slots_.size()];
        finalize_slot(s);  // frees the slot (waits for the frame that used it last)
        if (!src_pinned && !s.h_faces) CK(cudaMallocHost(&s.h_faces, slot_face_bytes_));
        if (!direct && !s.h_out) CK(cudaMallocHost(&s.h_out, slot_out_bytes_));
        // Only what the lens looks at is uploaded: plates with display != 0 (:764-766), and of
        // those only the texel rectangle the lensmap samples.  (TMA boxes may overhang the
        // rectangle; those texels are staged but never referenced by an entry.)
        const uint8_t *src = faces_host + static_cast<size_t>(f) * face_stride;
        cudaMemcpy3DBatchOp ops[BLINKY_MAX_PLATES];
        size_t nops = 0;
        for (int pl = 0; pl < g.numplates; ++pl) {
            if (!g.display[pl]) continue;
            const int *r = g.plate_rect[pl];
            if (r[0] > r[2] || r[1] > r[3]) continue;
            const size_t rw = static_cast<size_t>(r[2] - r[0] + 1), rh = static_cast<size_t>(r[3] - r[1] + 1);
            const size_t off = pl * ps2 + static_cast<size_t>(r[1]) * ps + r[0];   // in the dense device copy
            const uint8_t *from = src + (layout ? lay.plate_base[pl] + static_cast<size_t>(r[1]) * src_pitch + r[0] : off);
            size_t pitch = src_pitch;
            if (!src_pinned) {
                uint8_t *stage = s.h_faces + off;
                for (size_t y = 0; y < rh; ++y) memcpy(stage + y * ps, from + y * src_pitch, rw);
                from = stage;
                pitch = ps;
            }
            // a full-width rectangle of dense rows is one contiguous run: copy it as such
            const bool contiguous = rw == ps && pitch == rw;
            const size_t row = contiguous ? rw * rh : ps, rows = contiguous ? 1 : rh;
            cudaMemcpy3DBatchOp &op = ops[nops++];
            memset(&op, 0, sizeof op);
            op.src.type = cudaMemcpyOperandTypePointer;
            op.src.op.ptr.ptr = const_cast<uint8_t *>(from);
            op.src.op.ptr.rowLength = contiguous ? row : pitch;
            op.src.op.ptr.layerHeight = rows;
            op.dst.type = cudaMemcpyOperandTypePointer;
            op.dst.op.ptr.ptr = s.d_faces.as<uint8_t>() + off;
            op.dst.op.ptr.rowLength = row;
            op.dst.op.ptr.layerHeight = rows;
            op.extent = make_cudaExtent(contiguous ? rw * rh : rw, rows, 1);
            op.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
        }
        // all rectangles of the frame in ONE driver call (no gap between the DMA operations)
        size_t fail_idx = 0;
        if (nops > 0 && batch_copies_ && cudaMemcpy3DBatchAsync(nops, ops, &fail_idx, 0, s.stream) != cudaSuccess) {
            cudaGetLastError();  // not available on this driver: one copy per rectangle, from now on
            batch_copies_ = false;
        }
        for (size_t k = 0; !batch_copies_ && k < nops && ok; ++k) {
            const cudaError_t e = cudaMemcpy2DAsync(ops[k].dst.op.ptr.ptr, ops[k].dst.op.ptr.rowLength, ops[k].src.op.ptr.ptr, ops[k].src.op.ptr.rowLength,
                                                    ops[k].extent.width, ops[k].extent.height, cudaMemcpyHostToDevice, s.stream);
            if (e != cudaSuccess) ok = fail("cudaMemcpy2DAsync(H2D faces)", e);
        }
        if (!ok) break;
        s.dst = c.view + static_cast<size_t>(f) * r.out_stride;
        WarpRequest frame_r(s.d_faces.get(), slot_face_bytes_, s.d_out.get(), slot_out_bytes_, 1, s.stream);
        frame_r.dense_faces = true;   // the device copy is dense whatever the face layout
        if (!warp(frame_r)) { ok = false; break; }
        s.dst_rowbytes = dst_rowbytes;
        s.keep_unmapped = keep_unmapped;
        s.direct = direct;
        uint8_t *to = s.dst;
        cudaError_t e = !direct              ? cudaMemcpyAsync(s.h_out, s.d_out.get(), frame, cudaMemcpyDeviceToHost, s.stream)
                        : dst_rowbytes == W ? cudaMemcpyAsync(to, s.d_out.get(), frame, cudaMemcpyDeviceToHost, s.stream)
                                            : cudaMemcpy2DAsync(to, static_cast<size_t>(dst_rowbytes), s.d_out.get(), static_cast<size_t>(W),
                                                                static_cast<size_t>(W), static_cast<size_t>(H), cudaMemcpyDeviceToHost, s.stream);
        if (e != cudaSuccess) { ok = fail("cudaMemcpyAsync(D2H frame)", e); break; }
        e = cudaEventRecord(s.done, s.stream);
        if (e != cudaSuccess) { ok = fail("cudaEventRecord", e); break; }
        s.busy = true;
    }
    // drain in submission order
    for (size_t k = 0; k < slots_.size(); ++k) {
        Slot &s = *slots_[(static_cast<size_t>(f) + k) % slots_.size()];
        finalize_slot(s);
    }
    if (ok) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) ok = fail("warp_host", e);
    }
    return ok;
}

bool WarpDevice::alloc_device(size_t bytes, void **out) {
    CK(cudaSetDevice(device_));
    CK(cudaMalloc(out, bytes));
    return true;
}

bool WarpDevice::free_device(void *p) {
    CK(cudaSetDevice(device_));
    CK(cudaFree(p));
    return true;
}

bool WarpDevice::ipc_export(void *p, unsigned char handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    CK(cudaSetDevice(device_));
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, p));
    memcpy(handle, &h, 64);
    return true;
}

bool WarpDevice::ipc_open(const unsigned char handle[64], void **out) {
    CK(cudaSetDevice(device_));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    CK(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));  // maps the peer GPU's memory over NVLink
    return true;
}

bool WarpDevice::ipc_close(void *p) {
    CK(cudaSetDevice(device_));
    CK(cudaIpcCloseMemHandle(p));
    return true;
}

bool WarpDevice::alloc_pinned(size_t bytes, void **out) {
    CK(cudaSetDevice(device_));
    CK(cudaMallocHost(out, bytes));
    return true;
}

bool WarpDevice::free_pinned(void *p) {
    CK(cudaFreeHost(p));
    return true;
}

bool WarpDevice::sync() {
    CK(cudaSetDevice(device_));
    CK(cudaDeviceSynchronize());
    return true;
}

}  // namespace blinky
