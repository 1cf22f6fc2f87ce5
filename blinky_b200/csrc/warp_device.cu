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
#include "tile_plan.h"

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
    const uint32_t *rgba;       // [256] palette expansion table (RGBA mode)
    void *out;                  // frame 0
    size_t out_stride;          // bytes between frames
    uint32_t nquads;            // ceil(W*H / 4)
    uint32_t npix;              // W*H
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

// --------------------------------------------------------------------------
// K1: direct gather.  grid = (ceil(nquads/1024), nframes), block = 256.
// Thread t of CTA b owns quads b*1024 + c*256 + t, c = 0..3, so each of the
// four 128-bit lensmap loads of a warp covers 512 contiguous bytes and each
// 32-bit output store of a warp covers 128 contiguous bytes.
// --------------------------------------------------------------------------
template <bool RUBIX, bool RGBA>
__global__ void __launch_bounds__(kThreads) warp_gather_kernel(const WarpParams p) {
    __shared__ uint8_t s_lut[RUBIX ? 6 * 256 : 4];
    __shared__ uint32_t s_rgba[RGBA ? 256 : 1];
    if (RUBIX) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.lut);
        uint32_t *dst = reinterpret_cast<uint32_t *>(s_lut);
        for (int i = threadIdx.x; i < 6 * 256 / 4; i += kThreads) dst[i] = __ldg(src + i);
    }
    if (RGBA) {
        for (int i = threadIdx.x; i < 256; i += kThreads) s_rgba[i] = __ldg(p.rgba + i);
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
            if (ent[k] & BLINKY_LM_VALID) v[c][k] = ld_face(faces + (ent[k] & BLINKY_LM_INDEX_MASK));
        }
    }

#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
        const uint32_t q = q0 + c * kThreads;
        if (q >= p.nquads) continue;
        const uint32_t ent[4] = {e[c].x, e[c].y, e[c].z, e[c].w};
        const uint32_t all_valid = ent[0] & ent[1] & ent[2] & ent[3] & BLINKY_LM_VALID;
        uint32_t bgw = 0;
        if (!all_valid) bgw = __ldg(p.bg32 + q);
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
        if (RGBA) {
            uint4 w = make_uint4(s_rgba[px[0]], s_rgba[px[1]], s_rgba[px[2]], s_rgba[px[3]]);
            uint4 *o = reinterpret_cast<uint4 *>(static_cast<uint8_t *>(p.out) + static_cast<size_t>(blockIdx.y) * p.out_stride);
            st_stream_v4(o + q, w);
        } else {
            uint32_t w = px[0] | (px[1] << 8) | (px[2] << 16) | (px[3] << 24);
            uint32_t *o = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(p.out) + static_cast<size_t>(blockIdx.y) * p.out_stride);
            st_stream_u32(o + q, w);
        }
    }
}

// --------------------------------------------------------------------------
// K0: scalar kernel, one pixel per thread, byte stores.  Used only when the
// frame size or the caller's pointers rule out 32-bit stores (W*H % 4 != 0 or
// unaligned strides) — a correctness path for ragged sizes, not a fast path.
// --------------------------------------------------------------------------
template <bool RUBIX, bool RGBA>
__global__ void __launch_bounds__(kThreads) warp_scalar_kernel(const WarpParams p) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= p.npix) return;
    const uint32_t ent = __ldg(reinterpret_cast<const uint32_t *>(p.lensmap4) + i);
    const uint8_t *faces = p.faces + static_cast<size_t>(blockIdx.y) * p.face_stride;
    uint32_t b;
    if (ent & BLINKY_LM_VALID) {
        b = ld_face(faces + (ent & BLINKY_LM_INDEX_MASK));
        if (RUBIX) {
            const uint32_t t = (ent >> BLINKY_LM_TINT_SHIFT) & 7u;
            if (t != BLINKY_LM_TINT_NONE) b = __ldg(p.lut + t * 256 + b);
        }
    } else {
        b = __ldg(reinterpret_cast<const uint8_t *>(p.bg32) + i);
    }
    uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(blockIdx.y) * p.out_stride;
    if (RGBA) reinterpret_cast<uint32_t *>(o)[i] = __ldg(p.rgba + b);
    else o[i] = static_cast<uint8_t>(b);
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
    void *out;
    size_t out_stride;
    uint32_t *ticket;       // monotonic counter (never reset: see launch_ring)
    uint32_t ticket_base;   // its value when this launch starts
    uint32_t nstatic;       // units per warp that are assigned statically (warp w owns w, w+NW, ...) before it draws tickets
    uint32_t nbox, ngather, ntiles;
    uint32_t nframes, fchunk, nchunks, nunits;
    uint32_t ring_bytes;    // the warp's staging ring: boxes are packed into it one behind the other (multiple of 128)
    uint32_t max_inflight;  // boxes a warp keeps in flight at most (<= kRingBoxes)
    uint32_t ring_grid;     // CTAs [0, ring_grid) are ring warps, the CTAs behind them take one gather item each
    int width, height;
    uint32_t zero;  // always 0, but only the host knows: see stage_dep()
    uint32_t lab_bytes;  // (lab bit 5) bytes of box shape 0
    uint32_t lab;   // BLINKY_LAB builds only (make lab): bit 0 no stores, bit 1 bank-conflict-free gather offsets,
                    // bit 2 each warp-level store covers 128 contiguous bytes, bit 3 every frame reads frame 0's
                    // faces (L2-resident), bit 4 no box loads at all — wrong pixels, timing experiments
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

#ifdef BLINKY_LAB
#define LAB_ST8(POL)                                                                                                        \
    asm volatile("st.global" POL ".u32 [%0], %8;\n\tst.global" POL ".u32 [%1], %9;\n\tst.global" POL ".u32 [%2], %10;\n\t"    \
                 "st.global" POL ".u32 [%3], %11;\n\tst.global" POL ".u32 [%4], %12;\n\tst.global" POL ".u32 [%5], %13;\n\t"  \
                 "st.global" POL ".u32 [%6], %14;\n\tst.global" POL ".u32 [%7], %15;"                                        \
                 ::"l"(a[0]), "l"(a[1]), "l"(a[2]), "l"(a[3]), "l"(a[4]), "l"(a[5]), "l"(a[6]), "l"(a[7]), "r"(w[0]), "r"(w[1]), \
                   "r"(w[2]), "r"(w[3]), "r"(w[4]), "r"(w[5]), "r"(w[6]), "r"(w[7]) : "memory")
// store cache policy experiment: 0 .cs (shipped), 1 default (.wb), 2 .cg, 3 .wt
__device__ __forceinline__ void st_lab_u32x8(const uint64_t (&a)[8], const uint32_t (&w)[8], uint32_t pol) {
    if (pol == 1) LAB_ST8("");
    else if (pol == 2) LAB_ST8(".cg");
    else if (pol == 3) LAB_ST8(".wt");
    else LAB_ST8(".cs");
}
#endif

// ---- gather role of the ring kernel's launch ---------------------------------------------------------------
// GATHER tiles (plate seams, singular points, boxes too large to stage) read the globe directly: 32-bit
// entries, lane = column, so one warp-level load covers 32 consecutive screen pixels of one row.  They are
// bound by load latency, so they get plain parallelism: one extra one-warp CTA per (tile, 8 of its rows, 4
// frames) behind the ring CTAs in the same grid.  The launch leaves shared memory for two of them per SM next
// to the resident ring warps, so this work runs beside the ring warps from the start and fills the slots they
// vacate at the end.
constexpr int kGatherRows = 8, kGatherFrames = 4;

template <bool RUBIX, bool RGBA>
__device__ __forceinline__ void gather_item(const RingParams &p, uint32_t item, uint32_t lane) {
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
    uint32_t v[kGatherFrames][kGatherRows];
#pragma unroll
    for (int g = 0; g < kGatherFrames; ++g) {
        const uint32_t f = f0 + g;
        const uint8_t *__restrict__ faces = p.faces + static_cast<size_t>(f < f1 ? f : f0) * p.face_stride;
#pragma unroll
        for (int j = 0; j < kGatherRows; ++j) {
            v[g][j] = 0x100u;   // "take the background"
            if (e[j] & BLINKY_LM_VALID) v[g][j] = ld_face(faces + (e[j] & BLINKY_LM_INDEX_MASK));
        }
    }
#pragma unroll
    for (int j = 0; j < kGatherRows; ++j) {
        const uint32_t y = tile_y + j;
        if (y >= height) break;
        const size_t pix = static_cast<size_t>(y) * width + x;
        uint32_t bgv = 0, t = BLINKY_LM_TINT_NONE;
        if (!(e[j] & BLINKY_LM_VALID)) bgv = __ldg(p.bg + pix);
        else if (RUBIX) t = (e[j] >> BLINKY_LM_TINT_SHIFT) & 7u;
#pragma unroll
        for (int g = 0; g < kGatherFrames; ++g) {
            if (f0 + g >= f1) break;
            uint32_t b = v[g][j] & 0x100u ? bgv : v[g][j];
            if (RUBIX && t != BLINKY_LM_TINT_NONE) b = __ldg(p.lut + t * 256 + b);
            uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(f0 + g) * p.out_stride;
            if (RGBA) reinterpret_cast<uint32_t *>(o)[pix] = __ldg(p.rgba + b);
            else o[pix] = static_cast<uint8_t>(b);
        }
    }
}

// MINB: CTAs per SM the register allocation is sized for (ring warps plus the gather CTAs beside them)
template <bool RUBIX, bool RGBA, int MINB>
__global__ void __launch_bounds__(32, MINB) warp_ring_kernel(const __grid_constant__ RingParams p, const __grid_constant__ RingTmaps tm) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // XOR with a parameter that is always zero: keeps ptxas from re-reading the special register
    // (S2R, tens of cycles) at every `lane == 0` test instead of holding the lane number in a register
    const uint32_t lane = threadIdx.x ^ p.zero;
    if (blockIdx.x >= p.ring_grid) {   // the CTAs behind the ring warps: one gather item each
        gather_item<RUBIX, RGBA>(p, blockIdx.x - p.ring_grid, lane);
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
    if (RGBA) {
        for (uint32_t i = lane; i < 256; i += 32) s_rgba[i] = __ldg(p.rgba + i);
    }
    __syncwarp();
    const uint32_t lut_base = smem_u32(s_lut);

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
    // a function of the launch alone (the host advances ticket_base by it).
    uint32_t k_next = 0;        // index of the next ticket of this warp
    bool last_good = true;
    auto draw_now = [&]() {     // the k_next-th ticket, waiting for the counter if it is a dynamic one
        uint32_t t = 0xffffffffu;
        if (k_next < p.nstatic) {
            t = blockIdx.x + k_next * NW;
        } else if (last_good) {
            uint32_t d = 0;
            if (lane == 0) asm volatile("atom.global.add.u32 %0, [%1], 1;" : "=r"(d) : "l"(p.ticket) : "memory");
            t = p.nstatic * NW + (__shfl_sync(0xffffffffu, d, 0) - p.ticket_base);
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
                c_bytes = ((dz >> 16) & 0xffu) * (dz >> 24) * 128u;
#ifdef BLINKY_LAB
                if (p.lab & 32u) {   // every box through ONE descriptor (shape 0): is the TMA unit's descriptor cache the limit?
                    c_tmap = reinterpret_cast<uint64_t>(&tm.m[0]);
                    c_bytes = p.lab_bytes;
                }
#endif
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
#ifdef BLINKY_LAB
        if (lane == 0 && (c_entry || !(p.lab & 16u))) {
#else
        if (lane == 0) {
#endif
            const uint32_t bar = bars + 8 * is;
            mbar_expect_tx(bar, n);
            if (c_entry) bulk_load(ring + ipos + dep, p.entries + static_cast<size_t>(c_tile) * kBoxBlockBytes, n, bar);
#ifdef BLINKY_LAB
            else tma_load_box(ring + ipos + dep, reinterpret_cast<const CUtensorMap *>(c_tmap), c_bx, c_by, c_plate, (p.lab & 8u) ? 0 : static_cast<int>(c_frame), bar);
#else
            else tma_load_box(ring + ipos + dep, reinterpret_cast<const CUtensorMap *>(c_tmap), c_bx, c_by, c_plate, static_cast<int>(c_frame), bar);
#endif
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
            uint32_t a_bytes = ((A.dz >> 16) & 0xffu) * (A.dz >> 24) * 128u;   // size of this unit's boxes
#ifdef BLINKY_LAB
            if (p.lab & 32u) a_bytes = p.lab_bytes;
#endif
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
#ifdef BLINKY_LAB
            if (p.lab & 2u) {
#pragma unroll
                for (int i = 0; i < 32; ++i) off[i] = (lane * 4u + (i & 3) + (i >> 2) * 128u) & 1023u;
            }
#endif
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
            uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(A.f0) * p.out_stride + (static_cast<size_t>(qy) * width + qx) * opx;
            const uint32_t row4 = width * 4u * static_cast<uint32_t>(opx);   // four screen rows, bytes

            // one frame: wait for its box, 32 byte loads from shared memory, pack, hand the stage on
            auto gather_frame = [&](uint32_t (&w)[8]) {
#ifdef BLINKY_LAB
                if (!(p.lab & 16u))
#endif
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

            if (type == TILE_BOX_FULL) {
                for (uint32_t f = 0; f < A.nf; ++f) {
                    uint32_t w[8];
                    gather_frame(w);
                    if (RGBA) {
#pragma unroll
                        for (int q = 0; q < 8; ++q) store_rgba(o + static_cast<size_t>(static_cast<uint32_t>(q) * row4), w[q]);
                    } else {
                        uint64_t a[8];
#pragma unroll
                        for (int q = 0; q < 8; ++q) a[q] = reinterpret_cast<uint64_t>(o) + static_cast<uint64_t>(static_cast<uint32_t>(q) * row4);
#ifdef BLINKY_LAB
                        if (p.lab & 4u) {
                            uint8_t *fb = static_cast<uint8_t *>(p.out) + static_cast<size_t>(A.f0 + f) * p.out_stride + static_cast<size_t>(A.tile) * 1024u;
#pragma unroll
                            for (int q = 0; q < 8; ++q) a[q] = reinterpret_cast<uint64_t>(fb + q * 128 + lane * 4u);
                        }
                        if ((p.lab >> 8) & 3u) st_lab_u32x8(a, w, (p.lab >> 8) & 3u);
                        else if (!(p.lab & 1u) || w[0] == 0x12345679u)
#endif
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
                    if (qx < width && y < height) {
                        store_mask |= 1u << q;
                        if (m != 0xffffffffu) bgw[q] = __ldg(reinterpret_cast<const uint32_t *>(p.bg + static_cast<size_t>(y) * width + qx)) & ~m;
                    }
                }
                for (uint32_t f = 0; f < A.nf; ++f) {
                    uint32_t w[8];
                    gather_frame(w);
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        if (!((store_mask >> q) & 1u)) continue;
                        const uint32_t v = (w[q] & vmask[q]) | bgw[q];
                        uint8_t *dst = o + static_cast<size_t>(static_cast<uint32_t>(q) * row4);
                        if (RGBA) store_rgba(dst, v);
                        else st_stream_u32(reinterpret_cast<uint32_t *>(dst), v);
                    }
                    o += p.out_stride;
                }
            }
        } else {
            // ---- EMPTY: background only (quad layout)
            const uint32_t qx = tile_x + 4u * (lane & 7u), qy = tile_y + (lane >> 3);
            if (qx < width) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const uint32_t y = qy + 4u * q;
                    if (y >= height) break;
                    const size_t pix = static_cast<size_t>(y) * width + qx;
                    const uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(p.bg + pix));
                    for (uint32_t f = 0; f < A.nf; ++f) {
                        uint8_t *out_frame = static_cast<uint8_t *>(p.out) + static_cast<size_t>(A.f0 + f) * p.out_stride;
                        if (RGBA) st_stream_v4(reinterpret_cast<uint4 *>(out_frame) + (pix >> 2),
                                               make_uint4(s_rgba[v & 0xffu], s_rgba[(v >> 8) & 0xffu], s_rgba[(v >> 16) & 0xffu], s_rgba[v >> 24]));
                        else st_stream_u32(reinterpret_cast<uint32_t *>(out_frame) + (pix >> 2), v);
                    }
                }
            }
        }
        // rotate: A <- B <- C <- the ticket drawn above; the cursor moves with its unit
        uint32_t next_ticket = 0xffffffffu;
        if (k_next < p.nstatic) next_ticket = blockIdx.x + k_next * NW;
        else if (draw_dynamic) next_ticket = p.nstatic * NW + (__shfl_sync(0xffffffffu, drawn, 0) - p.ticket_base);
        ++k_next;
        last_good = next_ticket < p.nunits;
        A = B;
        B = C;
        C = describe(next_ticket);
        c_unit = c_unit > 0 ? c_unit - 1 : 0;
    }
}

// --------------------------------------------------------------------------
// K3: the GATHER tiles of plans in which they are many (more than kMergedGatherPercent of the tiles:
// minifying lenses, where a tile's texels do not fit a box), launched in front of the ring kernel; with
// few GATHER tiles they ride in the ring kernel's launch instead (gather_item).  Those tiles are bound
// by global-load latency and, at 32-byte sectors scattered over DRAM pages, by DRAM itself (ncu, 4K fisheye1:
// 4.6 TB/s = 70 % of the measured copy peak with about one useful byte in 20 fetched); they get plain parallelism: grid = (tiles, groups of 4 frames), 256 threads, a warp owns 4 tile rows and lane l is
// column l (one warp-level load = 32 consecutive screen pixels of one row).  The tile's entries are
// fetched once and reused for the frames of the group; all 16 gathers of a thread are issued before
// its first store.
// --------------------------------------------------------------------------
constexpr int kGatherFramesPerCta = 4;

template <bool RUBIX, bool RGBA>
__global__ void __launch_bounds__(kThreads) warp_tile_gather_kernel(const __grid_constant__ RingParams p, const uint32_t first_tile) {
    const uint32_t tid = threadIdx.x;
    const uint4 d = __ldg(reinterpret_cast<const uint4 *>(p.tiles + first_tile + blockIdx.x));
    const uint32_t type = (d.z >> 8) & kTileTypeMask;
    const uint32_t tile_x = d.w & 0xffffu, tile_y = d.w >> 16;
    const uint32_t width = static_cast<uint32_t>(p.width), height = static_cast<uint32_t>(p.height);
    const uint32_t f0 = blockIdx.y * kGatherFramesPerCta;
    const uint32_t f1 = min(f0 + kGatherFramesPerCta, p.nframes);

    if (type == TILE_EMPTY) {
        // quad layout: thread t copies 4 background pixels of row t/8
        const uint32_t x = tile_x + (tid & 7u) * 4u, y = tile_y + (tid >> 3);
        if (x >= width || y >= height) return;
        const size_t pix = static_cast<size_t>(y) * width + x;
        const uint32_t bgw = __ldg(reinterpret_cast<const uint32_t *>(p.bg + pix));
        const uint32_t px[4] = {bgw & 0xffu, (bgw >> 8) & 0xffu, (bgw >> 16) & 0xffu, bgw >> 24};
        for (uint32_t f = f0; f < f1; ++f) {
            uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(f) * p.out_stride;
            if (RGBA) st_stream_v4(reinterpret_cast<uint4 *>(o) + (pix >> 2), make_uint4(__ldg(p.rgba + px[0]), __ldg(p.rgba + px[1]), __ldg(p.rgba + px[2]), __ldg(p.rgba + px[3])));
            else st_stream_u32(reinterpret_cast<uint32_t *>(o) + (pix >> 2), bgw);
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
        if (!(e[j] & BLINKY_LM_VALID) && y < height) bgv[j] = __ldg(p.bg + static_cast<size_t>(y) * width + x);
    }
    uint32_t v[kGatherFramesPerCta][4];
#pragma unroll
    for (int g = 0; g < kGatherFramesPerCta; ++g) {
        const uint32_t f = f0 + g;
        const uint8_t *__restrict__ faces = p.faces + static_cast<size_t>(f < f1 ? f : f0) * p.face_stride;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            v[g][j] = bgv[j];
            if (e[j] & BLINKY_LM_VALID) v[g][j] = ld_face(faces + (e[j] & BLINKY_LM_INDEX_MASK));
        }
    }
#pragma unroll
    for (int g = 0; g < kGatherFramesPerCta; ++g) {
        const uint32_t f = f0 + g;
        if (f >= f1) break;
        uint8_t *o = static_cast<uint8_t *>(p.out) + static_cast<size_t>(f) * p.out_stride;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t y = tile_y + warp * 4 + j;
            if (y < height) {
                uint32_t b = v[g][j];
                if (RUBIX && (e[j] & BLINKY_LM_VALID)) {
                    const uint32_t t = (e[j] >> BLINKY_LM_TINT_SHIFT) & 7u;
                    if (t != BLINKY_LM_TINT_NONE) b = __ldg(p.lut + t * 256 + b);
                }
                const size_t pix = static_cast<size_t>(y) * width + x;
                if (RGBA) reinterpret_cast<uint32_t *>(o)[pix] = __ldg(p.rgba + b);
                else o[pix] = static_cast<uint8_t>(b);
            }
        }
    }
}

inline size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

}  // namespace

// ---------------------------------------------------------------------------
// frame pipeline slot
// ---------------------------------------------------------------------------
// ---- host -> device plate upload without the copy engine --------------------------------------
// The rectangles a lens samples are strided (e.g. half a plate wide); 2-D DMA copies of them reach
// ~35 GB/s here while the link does 45-48.  Pinned host memory is mapped into the device address
// space (UVA), so the SMs can pull exactly those bytes themselves, 16 bytes per thread.
struct UploadRects {
    int n;
    uint32_t off[6];     // byte offset of the rectangle's first 16-byte column in the frame
    uint32_t vec_w[6];   // rectangle width in 16-byte vectors
    uint32_t rows[6];
    uint32_t first[7];   // prefix sum of vec_w * rows
    uint32_t pitch;      // platesize
};

__global__ void __launch_bounds__(256) upload_rects_kernel(const uint8_t *__restrict__ host_src, uint8_t *__restrict__ dst, const __grid_constant__ UploadRects R) {
    const uint32_t total = R.first[R.n];
    for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < total; v += gridDim.x * blockDim.x) {
        int k = 0;
        while (v >= R.first[k + 1]) ++k;
        const uint32_t local = v - R.first[k];
        const uint32_t row = local / R.vec_w[k], col = local - row * R.vec_w[k];
        const size_t at = static_cast<size_t>(R.off[k]) + static_cast<size_t>(row) * R.pitch + static_cast<size_t>(col) * 16;
        const uint4 x = __ldcs(reinterpret_cast<const uint4 *>(host_src + at));
        *reinterpret_cast<uint4 *>(dst + at) = x;
    }
}

struct WarpDevice::Slot {
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    uint8_t *d_faces = nullptr, *d_out = nullptr;
    uint8_t *h_faces = nullptr, *h_out = nullptr;  // pinned staging
    bool busy = false;
    // finalize info
    uint8_t *dst = nullptr;          // first frame of the group
    size_t dst_frame_stride = 0;
    int nf = 0;                      // frames in the slot
    int dst_rowbytes = 0, x0 = 0, y0 = 0;
    bool keep_unmapped = false, direct = false;
};

struct WarpDevice::TmapSet {   // host-side: the descriptors travel in the kernel's parameter block
    const void *faces = nullptr;
    size_t face_stride = 0;
    int nframes = 0;
    RingTmaps table;
    uint64_t last_use = 0;
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

#define CK(call)                                      \
    do {                                              \
        cudaError_t e_ = (call);                      \
        if (e_ != cudaSuccess) return fail(#call, e_); \
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
    smem_per_sm_ = prop.sharedMemPerMultiprocessor;
    if (const char *e = getenv("BLINKY_E2E_UPLOAD")) upload_by_kernel_ = strcmp(e, "kernel") == 0;
    if (const char *e = getenv("BLINKY_E2E_OUT")) out_by_kernel_ = strcmp(e, "direct") == 0;
    if (const char *e = getenv("BLINKY_E2E_BATCH")) batch_copies_ = atoi(e) != 0;
    if (const char *e = getenv("BLINKY_RING_BYTES")) ring_bytes_override_ = atoi(e);
    if (const char *e = getenv("BLINKY_RING_BOXES")) ring_boxes_ = atoi(e);
    if (const char *e = getenv("BLINKY_MERGED_ITEMS")) merged_items_max_ = atoi(e);
    if (const char *e = getenv("BLINKY_RING_CTAS")) ring_ctas_cap_ = atoi(e);
    if (const char *e = getenv("BLINKY_FCHUNK")) fchunk_ = atoi(e);
    if (const char *e = getenv("BLINKY_SERIAL_GATHER")) serial_gather_ = atoi(e) != 0;  // GATHER tiles in their own kernel before the ring kernel (A/B)
    if (const char *e = getenv("BLINKY_STATIC_PCT")) static_pct_ = std::max(0, std::min(100, atoi(e)));
    if (const char *e = getenv("BLINKY_L2_PROMOTION")) l2_promotion_ = atoi(e) & 3;  // 0 none, 1 64 B, 2 128 B, 3 256 B
    cudaStream_t s;
    e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaStreamCreate: ") + cudaGetErrorString(e));
    stream_ = s;
    e = cudaMalloc(&d_lut_, 6 * 256);
    if (e == cudaSuccess) e = cudaMemset(d_lut_, 0, 6 * 256);
    if (e == cudaSuccess) e = cudaMalloc(&d_rgba_, 256 * 4);
    if (e == cudaSuccess) e = cudaMemset(d_rgba_, 0, 256 * 4);
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaMalloc: ") + cudaGetErrorString(e));
}

WarpDevice::~WarpDevice() {
    cudaSetDevice(device_);
    cudaDeviceSynchronize();
    for (Slot *s : slots_) {
        if (s->stream) cudaStreamDestroy(s->stream);
        if (s->done) cudaEventDestroy(s->done);
        cudaFree(s->d_faces);
        cudaFree(s->d_out);
        if (s->h_faces) cudaFreeHost(s->h_faces);
        if (s->h_out) cudaFreeHost(s->h_out);
        delete s;
    }
    cudaFree(d_lensmap_);
    cudaFree(d_lut_);
    cudaFree(d_bg_);
    cudaFree(d_rgba_);
    cudaFree(d_tiles_);
    cudaFree(d_entries_);
    for (TmapSet *t : tmap_sets_) delete t;
    for (TicketCounter &c : tickets_) cudaFree(c.d_counter);
    if (stream_) cudaStreamDestroy(static_cast<cudaStream_t>(stream_));
}

bool WarpDevice::upload_lensmap(const LensmapUpload &lm) {
    CK(cudaSetDevice(device_));
    CK(cudaDeviceSynchronize());  // nothing may still be reading the old map
    const size_t npix = static_cast<size_t>(lm.width) * lm.height;
    const size_t npad = round_up(npix, kPixelsPerBlock);
    if (npad != npix_pad_) {
        cudaFree(d_lensmap_);
        cudaFree(d_bg_);
        d_lensmap_ = nullptr;
        d_bg_ = nullptr;
        CK(cudaMalloc(&d_lensmap_, npad * sizeof(uint32_t)));
        CK(cudaMalloc(&d_bg_, npad));
        CK(cudaMemset(d_bg_, 0, npad));
    } else if (lm.width != width_ || lm.height != height_) {
        CK(cudaMemset(d_bg_, 0, npad));
    }
    // padding entries are "unmapped"
    CK(cudaMemset(d_lensmap_, 0, npad * sizeof(uint32_t)));
    CK(cudaMemcpy(d_lensmap_, lm.packed, npix * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_lut_, lm.palmaps, 6 * 256, cudaMemcpyHostToDevice));
    width_ = lm.width;
    height_ = lm.height;
    platesize_ = lm.platesize;
    numplates_ = lm.numplates;
    npix_ = npix;
    npix_pad_ = npad;
    rubix_ = lm.rubix;
    memcpy(display_, lm.display, sizeof display_);
    memcpy(plate_rect_, lm.plate_rect, sizeof plate_rect_);
    span_off_.assign(lm.span_off, lm.span_off + lm.height + 1);
    spans_.assign(lm.spans, lm.spans + lm.nspans * 2);
    have_lensmap_ = true;
    // tiled layout
    have_plan_ = false;
    plan_has_box_ = false;
    cudaFree(d_tiles_);
    cudaFree(d_entries_);
    d_tiles_ = nullptr;
    d_entries_ = nullptr;
    for (TmapSet *t : tmap_sets_) delete t;
    tmap_sets_.clear();
    if (lm.plan && !lm.plan->tiles.empty()) {
        const TilePlan &pl = *lm.plan;
        CK(cudaMalloc(&d_tiles_, pl.tiles.size() * sizeof(TileDesc)));
        CK(cudaMemcpy(d_tiles_, pl.tiles.data(), pl.tiles.size() * sizeof(TileDesc), cudaMemcpyHostToDevice));
        CK(cudaMalloc(&d_entries_, pl.entries.size()));
        CK(cudaMemcpy(d_entries_, pl.entries.data(), pl.entries.size(), cudaMemcpyHostToDevice));
        ntiles_ = static_cast<uint32_t>(pl.tiles.size());
        nbox_tiles_ = static_cast<uint32_t>(pl.n_box);
        ngather_tiles_ = static_cast<uint32_t>(pl.n_gather);
        stage_bytes_ = pl.stage_bytes;
        shapes_ = pl.shapes;
        plan_has_box_ = pl.n_box > 0;
        have_plan_ = true;
        char buf[256];
        snprintf(buf, sizeof buf, "tiles %dx%d of %dx%d px: %d box (TMA, %.2f B/px staged), %d gather, %d empty; entries %.2f B/px",
                 pl.tiles_x, pl.tiles_y, kTileW, kTileH, pl.n_box, static_cast<double>(pl.box_bytes) / static_cast<double>(npix),
                 pl.n_gather, pl.n_empty, static_cast<double>(pl.entries.size()) / static_cast<double>(npix));
        plan_summary_ = buf;
    }
    // frame slots depend on the sizes: rebuild lazily
    for (Slot *s : slots_) {
        cudaStreamDestroy(s->stream);
        cudaEventDestroy(s->done);
        cudaFree(s->d_faces);
        cudaFree(s->d_out);
        cudaFreeHost(s->h_faces);
        cudaFreeHost(s->h_out);
        delete s;
    }
    slots_.clear();
    return true;
}

bool WarpDevice::set_background(const uint8_t *bg_host) {
    if (!have_lensmap_) {
        err_ = "set_background: build a lensmap first (the background has the view's size)";
        return false;
    }
    CK(cudaSetDevice(device_));
    CK(cudaDeviceSynchronize());
    if (bg_host) CK(cudaMemcpy(d_bg_, bg_host, npix_, cudaMemcpyHostToDevice));
    else CK(cudaMemset(d_bg_, 0, npix_pad_));
    return true;
}

bool WarpDevice::set_rgba_table(const uint32_t table[256]) {
    CK(cudaSetDevice(device_));
    CK(cudaMemcpy(d_rgba_, table, 256 * 4, cudaMemcpyHostToDevice));
    have_rgba_ = true;
    return true;
}

bool WarpDevice::warp(const void *d_faces, size_t face_stride, void *d_out, size_t out_stride, int nframes, void *stream,
                      bool rgba) {
    if (!have_lensmap_) {
        err_ = "warp: no lensmap on the device (call blinky_build_lensmap)";
        return false;
    }
    if (nframes <= 0) return true;
    if (nframes > 65535) {
        err_ = "warp: at most 65535 frames per launch";
        return false;
    }
    const size_t opx = rgba ? 4 : 1;
    if (rgba && (reinterpret_cast<uintptr_t>(d_out) % 4 != 0 || (nframes > 1 && out_stride % 4 != 0))) {
        err_ = "warp (RGBA): the output buffer and the frame stride must be 4-byte aligned";
        return false;
    }
    // the tiled kernel writes 4-pixel words at (y*W + x): needs W % 4 == 0 and aligned frames
    const bool tiled_ok = have_plan_ && (width_ % 4 == 0) && (reinterpret_cast<uintptr_t>(d_out) % (4 * opx) == 0) &&
                          (out_stride % (4 * opx) == 0 || nframes == 1) &&
                          (!plan_has_box_ || (reinterpret_cast<uintptr_t>(d_faces) % 16 == 0 && (face_stride % 16 == 0 || nframes == 1)));
    if (variant_ == BLINKY_KERNEL_GATHER || !tiled_ok) return launch_flat(d_faces, face_stride, d_out, out_stride, nframes, stream, rgba);
    return launch_ring(d_faces, face_stride, d_out, out_stride, nframes, stream, rgba);
}

WarpDevice::TmapSet *WarpDevice::get_tmaps(const void *d_faces, size_t face_stride, int nframes) {
    const uint64_t tick = ++tmap_tick_;
    for (TmapSet *t : tmap_sets_)
        if (t->faces == d_faces && t->face_stride == face_stride && t->nframes == nframes) {
            t->last_use = tick;
            return t;
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
        t = tmap_sets_[0];
        for (TmapSet *c : tmap_sets_)
            if (c->last_use < t->last_use) t = c;
    } else {
        t = new TmapSet();
        tmap_sets_.push_back(t);
    }
    t->faces = d_faces;
    t->face_stride = face_stride;
    t->nframes = nframes;
    t->last_use = tick;
    memset(&t->table, 0, sizeof t->table);
    const cuuint64_t ps = static_cast<cuuint64_t>(platesize_);
    // 4-D view of the globe: (x, y, plate, frame)
    const cuuint64_t dims[4] = {ps, ps, static_cast<cuuint64_t>(numplates_), static_cast<cuuint64_t>(nframes)};
    const cuuint64_t fstride = nframes > 1 ? static_cast<cuuint64_t>(face_stride) : ps * ps * static_cast<cuuint64_t>(numplates_);
    const cuuint64_t strides[3] = {ps, ps * ps, fstride};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    for (size_t si = 0; si < shapes_.size() && si < static_cast<size_t>(kMaxShapes); ++si) {
        const uint32_t w16 = shapes_[si] >> 8, h8 = shapes_[si] & 0xff;
        cuuint32_t box[4] = {w16 * 16, h8 * 8, 1, 1};
#ifdef BLINKY_LAB
        // timing experiment: the same bytes as wider, flatter boxes (fewer TMA rows; wrong texels)
        if (const char *e = getenv("BLINKY_LAB_FLAT")) {
            for (int k = atoi(e); k > 1; k /= 2)
                if (box[0] * 2 <= 256 && box[1] % 2 == 0) box[0] *= 2, box[1] /= 2;
        }
#endif
        CUresult r = reinterpret_cast<EncodeTiledFn>(encode_fn_)(
            &t->table.m[si], CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void *>(d_faces), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, static_cast<CUtensorMapL2promotion>(l2_promotion_), CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            char buf[160];
            snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled(box %ux%u, ps %d) failed with CUresult %d", w16 * 16, h8 * 8, platesize_, static_cast<int>(r));
            err_ = buf;
            t->faces = nullptr;
            return nullptr;
        }
    }
    return t;
}

// CTAs per SM the ring kernel's register allocation is sized for: 16 (128 registers per thread; the BOX path uses 96,
// 116 with the rubix overlay).  How many ring warps are resident is decided in launch_ring.
template <bool RUBIX>
constexpr int ring_warps() { return 16; }
// Resident ring warps per SM by default (BLINKY_RING_CTAS): measured on the 4K panini batch (bench.py, H100 80GB HBM3
// at a 400 W power limit) 8 / 10 / 12 / 14 / 16 warps give 578 / 578 / 657 / 652 / 653 Gpixel/s — beyond 12, more
// warps only spread the faces' L2 footprint; the registers left over go to the gather CTAs.
constexpr int kRingWarpsDefault = 12;
// GATHER tiles ride in the ring kernel's launch (gather_item) while they are at most this share of the plan; beyond
// it (minifying lenses: thousands of GATHER tiles) the 256-thread gather kernel K3 in front of the ring kernel is
// faster than tens of thousands of one-warp CTAs.
constexpr uint32_t kMergedGatherPercent = 5;

template <bool RUBIX, bool RGBA>
static cudaError_t ring_config(size_t smem, int *ctas_per_sm) {
    cudaError_t e = cudaFuncSetAttribute(warp_ring_kernel<RUBIX, RGBA, ring_warps<RUBIX>()>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, warp_ring_kernel<RUBIX, RGBA, ring_warps<RUBIX>()>, 32, smem);
}

static cudaError_t ring_config_v(bool rubix, bool rgba, size_t smem, int *n) {
    return rubix && rgba ? ring_config<true, true>(smem, n)
           : rubix       ? ring_config<true, false>(smem, n)
           : rgba        ? ring_config<false, true>(smem, n)
                         : ring_config<false, false>(smem, n);
}

static void ring_launch_v(bool rubix, bool rgba, uint32_t grid, size_t smem, cudaStream_t st, const RingParams &p, const RingTmaps &tm) {
    if (rubix && rgba) warp_ring_kernel<true, true, ring_warps<true>()><<<grid, 32, smem, st>>>(p, tm);
    else if (rubix) warp_ring_kernel<true, false, ring_warps<true>()><<<grid, 32, smem, st>>>(p, tm);
    else if (rgba) warp_ring_kernel<false, true, ring_warps<false>()><<<grid, 32, smem, st>>>(p, tm);
    else warp_ring_kernel<false, false, ring_warps<false>()><<<grid, 32, smem, st>>>(p, tm);
}

bool WarpDevice::launch_ring(const void *d_faces, size_t face_stride, void *d_out, size_t out_stride, int nframes,
                             void *stream, bool rgba) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RingParams p;
    p.tiles = static_cast<const TileDesc *>(d_tiles_);
    p.entries = d_entries_;
    static const RingTmaps kNoTmaps = {};
    const RingTmaps *tm = &kNoTmaps;
    if (plan_has_box_) {
        TmapSet *t = get_tmaps(d_faces, face_stride, nframes);
        if (!t) return false;
        tm = &t->table;
    }
    p.faces = static_cast<const uint8_t *>(d_faces);
    p.face_stride = face_stride;
    p.bg = d_bg_;
    p.lut = d_lut_;
    p.rgba = d_rgba_;
    p.out = d_out;
    p.out_stride = out_stride;
    p.nbox = nbox_tiles_;
    p.ngather = ngather_tiles_;
    p.ntiles = ntiles_;
    p.nframes = static_cast<uint32_t>(nframes);
    p.width = width_;
    p.height = height_;
    p.zero = 0;
    p.lab = 0;
    if (const char *e = getenv("BLINKY_LAB")) p.lab = static_cast<uint32_t>(atoi(e));
    p.lab_bytes = shapes_.empty() ? 128u : static_cast<uint32_t>((shapes_[0] >> 8) * (shapes_[0] & 0xff) * 128);
    const bool rubix = rubix_;
    const int vi = (rubix ? 1 : 0) | (rgba ? 2 : 0);
    // The ring kernel takes the BOX tiles [0, nbox) and the EMPTY tiles; the GATHER tiles in between go to the
    // gather kernel K3 on the context's side stream (forked from and joined to the caller's stream), so the two
    // kernels share the GPU instead of queueing behind each other.
    const uint32_t nempty = ntiles_ - nbox_tiles_ - ngather_tiles_;
    const uint32_t ring_tiles = nbox_tiles_ + nempty;
    // Ring geometry: as many warps per SM as the registers allow (or BLINKY_RING_CTAS), each with the largest
    // staging ring that still lets that many CTAs share the SM's shared memory; fewer warps if the plan's
    // largest box would not fit such a ring.
    const size_t fixed = kRingBarBytes + (rubix ? 6 * 256 : 0) + (rgba ? 1024 : 0);
    const uint32_t max_box = std::max<uint32_t>(static_cast<uint32_t>(stage_bytes_ > 0 ? stage_bytes_ : 128), kBoxBlockBytes);  // largest ring item
    // (few gather items in absolute terms — short launches — also ride along: a second kernel launch costs more than they do)
    const uint32_t all_gather_items = ngather_tiles_ * (kTileH / kGatherRows) * static_cast<uint32_t>((nframes + kGatherFrames - 1) / kGatherFrames);
    const bool merged_gather = !serial_gather_ && ngather_tiles_ > 0 &&
                               (ngather_tiles_ * 100u <= ntiles_ * kMergedGatherPercent || all_gather_items <= static_cast<uint32_t>(merged_items_max_));
    int want = std::min(kRingWarpsDefault, rubix ? ring_warps<true>() : ring_warps<false>());
    if (ring_ctas_cap_ > 0) want = std::min(ring_ctas_cap_, rubix ? ring_warps<true>() : ring_warps<false>());
    // ring size: twice the plan's largest box plus an entry block (two boxes of any size and the next unit's entries in
    // flight), as far as `want`
    // resident warps — plus two gather CTAs, which
    // carry the same allocation, when GATHER tiles ride along — leave room in the SM's shared memory
    uint32_t ring_bytes = 0;
    for (; want >= 1; --want) {
        const size_t per_cta = smem_per_sm_ / static_cast<size_t>(want + (merged_gather ? 2 : 0));
        if (per_cta < 1024 + fixed + max_box) continue;
        const uint32_t room = static_cast<uint32_t>((per_cta - 1024 - fixed) / 128 * 128);
        ring_bytes = std::min(room, std::max(2u * max_box + kBoxBlockBytes, 8192u));
        if (ring_bytes_override_ > 0) ring_bytes = std::min(room, std::max<uint32_t>(max_box, static_cast<uint32_t>(ring_bytes_override_) / 128 * 128));
        break;
    }
    if (want < 1) {
        err_ = "ring kernel: the plan's largest box does not fit the staging ring";
        return false;
    }
    p.ring_bytes = ring_bytes;
    // items in flight per warp: two boxes and (at unit boundaries) the next entry block (BLINKY_RING_BOXES overrides)
    p.max_inflight = static_cast<uint32_t>(std::max(1, std::min(ring_boxes_ > 0 ? ring_boxes_ : 3, kRingBoxes)));
    const size_t smem = static_cast<size_t>(ring_bytes) + fixed;
    if (ring_ctas_per_sm_[vi] == 0 || ring_smem_[vi] != smem) {
        int n = 0;
        cudaError_t e = ring_config_v(rubix, rgba, smem, &n);
        if (e != cudaSuccess) return fail("ring kernel configuration (shared memory / occupancy)", e);
        if (n < 1) {
            err_ = "ring kernel does not fit on an SM";
            return false;
        }
        ring_ctas_per_sm_[vi] = n;
        ring_smem_[vi] = smem;
    }
    int ctas = std::min(ring_ctas_per_sm_[vi], want);
    uint32_t grid = static_cast<uint32_t>(sm_count_ * ctas);
    // frames per unit: a unit pays a fixed cost (entry unpack, ring refill across the boundary: ~0.8 frame
    // times) and the launch ends with a tail of about one unit; pick the chunk that minimises
    // units-per-warp x (chunk + 0.8) + chunk
    uint32_t fchunk = fchunk_ > 0 ? static_cast<uint32_t>(fchunk_) : 1;
    if (fchunk_ <= 0) {
        double best = 0;
        for (uint32_t c = 1; c <= std::min<uint32_t>(p.nframes, 16u); ++c) {
            const double units = static_cast<double>(ring_tiles) * ((p.nframes + c - 1) / c);
            const double cost = std::max(1.0, units / grid) * (c + 0.8) + c;
            if (c == 1 || cost < best) best = cost, fchunk = c;
        }
    }
    if (fchunk > p.nframes) fchunk = p.nframes;
    p.fchunk = fchunk;
    p.nchunks = (p.nframes + fchunk - 1) / fchunk;
    p.nunits = ring_tiles * p.nchunks;
    if (grid > p.nunits) grid = p.nunits;
    char buf[640];
    int nbuf = 0;
    // GATHER tiles: one-warp CTAs behind the ring warps in the same grid (see gather_item); only a plan without BOX and
    // EMPTY tiles launches the stand-alone gather kernel.
    uint32_t ngather = ngather_tiles_;
#ifdef BLINKY_LAB
    if (getenv("BLINKY_LAB_NOK3")) ngather = 0;  // time the ring warps alone
#endif
    const uint32_t gather_items = ngather * (kTileH / kGatherRows) * static_cast<uint32_t>((nframes + kGatherFrames - 1) / kGatherFrames);
    buf[0] = 0;
    if (ngather > 0 && (grid == 0 || !merged_gather)) {
        dim3 g2(ngather, static_cast<unsigned>((nframes + kGatherFramesPerCta - 1) / kGatherFramesPerCta));
        if (rubix && rgba) warp_tile_gather_kernel<true, true><<<g2, kThreads, 0, st>>>(p, nbox_tiles_);
        else if (rubix) warp_tile_gather_kernel<true, false><<<g2, kThreads, 0, st>>>(p, nbox_tiles_);
        else if (rgba) warp_tile_gather_kernel<false, true><<<g2, kThreads, 0, st>>>(p, nbox_tiles_);
        else warp_tile_gather_kernel<false, false><<<g2, kThreads, 0, st>>>(p, nbox_tiles_);
        ++launches_;
        snprintf(buf, sizeof buf, "warp_tile_gather_kernel<rubix=%d,rgba=%d> grid=(%u,%u) block=%d", rubix, rgba, g2.x, g2.y, kThreads);
    }
    if (grid > 0) {
        // ticket counter of this stream (launches on one stream are serialised; the counter is never reset:
        // the kernel subtracts the value it had when the launch started)
        TicketCounter *tc = nullptr;
        for (TicketCounter &c : tickets_)
            if (c.stream == stream) tc = &c;
        if (!tc) {
            if (tickets_.size() >= 64) {  // streams come and go: start over
                CK(cudaDeviceSynchronize());
                for (TicketCounter &c : tickets_) cudaFree(c.d_counter);
                tickets_.clear();
            }
            TicketCounter c;
            c.stream = stream;
            c.base = 0;
            CK(cudaMalloc(&c.d_counter, sizeof(uint32_t)));
            CK(cudaMemsetAsync(c.d_counter, 0, sizeof(uint32_t), st));
            tickets_.push_back(c);
            tc = &tickets_.back();
        }
        p.ticket = tc->d_counter;
        p.ticket_base = tc->base;
        // static share of the schedule (see the kernel): static_pct_ percent of the units, whole rounds
        uint32_t nstatic = static_cast<uint32_t>(static_cast<uint64_t>(p.nunits) * static_cast<uint64_t>(static_pct_) / 100u / grid);
        p.nstatic = nstatic;
        // draws of this launch: every unit beyond the static ones is drawn exactly once, and every warp that
        // draws at all draws exactly one ticket past the end (it stops at its first bad ticket).  A warp draws
        // iff its last static ticket is good (all warps when there are no static rounds).
        const uint64_t nst = static_cast<uint64_t>(nstatic) * grid;
        const uint32_t good = p.nunits > nst ? static_cast<uint32_t>(p.nunits - nst) : 0u;
        uint32_t drawers = grid;
        if (nstatic > 0) {
            const uint64_t before_last = static_cast<uint64_t>(nstatic - 1) * grid;
            drawers = p.nunits > before_last ? static_cast<uint32_t>(std::min<uint64_t>(p.nunits - before_last, grid)) : 0u;
        }
        tc->base += good + drawers;

        p.ring_grid = grid;
        const uint32_t extra = merged_gather ? gather_items : 0u;
        ring_launch_v(rubix, rgba, grid + extra, smem, st, p, *tm);
        ++launches_;
        nbuf = static_cast<int>(strlen(buf));
        snprintf(buf + nbuf, sizeof buf - static_cast<size_t>(nbuf),
                 "%swarp_ring_kernel<rubix=%d,rgba=%d> grid=%u+%u block=32 (%d ring warps/SM, TMA box ring of %u B, <=%u boxes in flight, %u frames/unit, %u units; "
                 "%u gather CTAs of %dx32 px x %d frames)",
                 nbuf ? " + " : "", rubix, rgba, grid, extra, ctas, p.ring_bytes, p.max_inflight, fchunk, p.nunits, extra, kGatherRows, kGatherFrames);
    }
    last_kernel_ = buf;
    CK(cudaGetLastError());
    return true;
}

bool WarpDevice::launch_flat(const void *d_faces, size_t face_stride, void *d_out, size_t out_stride, int nframes, void *stream,
                             bool rgba) {
    // NULL is CUDA's default stream (what torch.cuda.current_stream() hands out
    // unless the caller made its own) — NOT this context's private stream.
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    WarpParams p;
    p.lensmap4 = reinterpret_cast<const uint4 *>(d_lensmap_);
    p.faces = static_cast<const uint8_t *>(d_faces);
    p.face_stride = face_stride;
    p.bg32 = reinterpret_cast<const uint32_t *>(d_bg_);
    p.lut = d_lut_;
    p.rgba = d_rgba_;
    p.out = d_out;
    p.out_stride = out_stride;
    p.nquads = static_cast<uint32_t>((npix_ + 3) / 4);
    p.npix = static_cast<uint32_t>(npix_);

    const size_t opx = rgba ? 4 : 1;  // output bytes per pixel
    const bool vector_ok = (npix_ % 4 == 0) && (reinterpret_cast<uintptr_t>(d_out) % (4 * opx) == 0) &&
                           (out_stride % (4 * opx) == 0 || nframes == 1);
    const bool rubix = rubix_;
    if (vector_ok) {
        dim3 grid(static_cast<unsigned>(npix_pad_ / kPixelsPerBlock), static_cast<unsigned>(nframes));
        if (rubix && rgba) warp_gather_kernel<true, true><<<grid, kThreads, 0, st>>>(p);
        else if (rubix) warp_gather_kernel<true, false><<<grid, kThreads, 0, st>>>(p);
        else if (rgba) warp_gather_kernel<false, true><<<grid, kThreads, 0, st>>>(p);
        else warp_gather_kernel<false, false><<<grid, kThreads, 0, st>>>(p);
        char buf[160];
        snprintf(buf, sizeof buf, "warp_gather_kernel<rubix=%d,rgba=%d> grid=(%u,%u) block=%d", rubix, rgba, grid.x, grid.y, kThreads);
        last_kernel_ = buf;
    } else {
        dim3 grid(static_cast<unsigned>((npix_ + kThreads - 1) / kThreads), static_cast<unsigned>(nframes));
        if (rubix && rgba) warp_scalar_kernel<true, true><<<grid, kThreads, 0, st>>>(p);
        else if (rubix) warp_scalar_kernel<true, false><<<grid, kThreads, 0, st>>>(p);
        else if (rgba) warp_scalar_kernel<false, true><<<grid, kThreads, 0, st>>>(p);
        else warp_scalar_kernel<false, false><<<grid, kThreads, 0, st>>>(p);
        char buf[160];
        snprintf(buf, sizeof buf, "warp_scalar_kernel<rubix=%d,rgba=%d> grid=(%u,%u) block=%d", rubix, rgba, grid.x, grid.y, kThreads);
        last_kernel_ = buf;
    }
    ++launches_;
    CK(cudaGetLastError());
    return true;
}

bool WarpDevice::ensure_slots() {
    if (!slots_.empty()) return true;
    int kSlots = 3;
    if (const char *e = getenv("BLINKY_HOST_SLOTS")) {  // pipeline depth of blinky_warp_host (experiments)
        const int v = atoi(e);
        if (v >= 1 && v <= 16) kSlots = v;
    }
    // A slot can hold a GROUP of frames (one batched upload, one launch, one copy back per group; BLINKY_HOST_GROUP).
    // Measured with 16-frame calls: 1 / 2 / 4 / 8 frames per group give 28.4 / 26.6 / 25.9 / 25.0 Gpx/s — fewer, larger
    // copies do not make the link faster, and the coarser pipeline overlaps less — so the default is one frame per slot.
    host_group_ = 1;
    if (const char *e = getenv("BLINKY_HOST_GROUP")) {
        const int v = atoi(e);
        if (v >= 1 && v <= kMaxHostGroup) host_group_ = v;
    }
    slot_face_bytes_ = static_cast<size_t>(numplates_) * platesize_ * platesize_;
    slot_out_bytes_ = round_up(npix_, 16);
    for (int i = 0; i < kSlots; ++i) {
        Slot *s = new Slot();
        slots_.push_back(s);
        CK(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&s->done, cudaEventDisableTiming));
        CK(cudaMalloc(&s->d_faces, slot_face_bytes_ * host_group_));
        CK(cudaMemset(s->d_faces, 0, slot_face_bytes_ * host_group_));
        CK(cudaMalloc(&s->d_out, slot_out_bytes_ * host_group_));
        // (pinned staging for callers whose buffers are not pinned: allocated when first needed)
    }
    return true;
}

void WarpDevice::finalize_slot(Slot &s) {
    if (!s.busy) return;
    cudaEventSynchronize(s.done);
    s.busy = false;
    if (s.direct) return;  // the copy engine already wrote the caller's buffer
    const int W = width_, H = height_;
    for (int k = 0; k < s.nf; ++k) {
        uint8_t *dst = s.dst + static_cast<size_t>(k) * s.dst_frame_stride + static_cast<size_t>(s.y0) * s.dst_rowbytes + s.x0;
        const uint8_t *frame = s.h_out + static_cast<size_t>(k) * slot_out_bytes_;
        if (s.keep_unmapped) {
            // only mapped pixels are written, like `if (*lmap)` in render_lensmap (:2413)
            for (int y = 0; y < H; ++y) {
                const uint8_t *src = frame + static_cast<size_t>(y) * W;
                uint8_t *row = dst + static_cast<size_t>(y) * s.dst_rowbytes;
                for (int32_t j = span_off_[static_cast<size_t>(y)]; j < span_off_[static_cast<size_t>(y) + 1]; ++j) {
                    const int32_t a = spans_[static_cast<size_t>(j) * 2], b = spans_[static_cast<size_t>(j) * 2 + 1];
                    memcpy(row + a, src + a, static_cast<size_t>(b - a));
                }
            }
        } else if (s.dst_rowbytes == W) {
            memcpy(dst, frame, static_cast<size_t>(W) * H);
        } else {
            for (int y = 0; y < H; ++y) memcpy(dst + static_cast<size_t>(y) * s.dst_rowbytes, frame + static_cast<size_t>(y) * W, static_cast<size_t>(W));
        }
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

bool WarpDevice::warp_host(const uint8_t *faces_host, size_t face_stride, uint8_t *dst_host, size_t dst_frame_stride,
                           int dst_rowbytes, int x0, int y0, int nframes, bool keep_unmapped) {
    if (!have_lensmap_) {
        err_ = "warp_host: no lensmap on the device (call blinky_build_lensmap)";
        return false;
    }
    CK(cudaSetDevice(device_));
    if (!ensure_slots()) return false;
    const size_t ps2 = static_cast<size_t>(platesize_) * platesize_;
    // (one driver query per distinct buffer, not two per call)
    if (faces_host != pin_src_ptr_) pin_src_ptr_ = faces_host, pin_src_ = is_pinned(faces_host);
    if (dst_host != pin_dst_ptr_) pin_dst_ptr_ = dst_host, pin_dst_ = is_pinned(dst_host);
    const bool src_pinned = pin_src_, dst_pinned = pin_dst_;
    const int W = width_, H = height_;
    bool ok = true;
    const int G = std::max(1, std::min(host_group_, kMaxHostGroup));
    int group = 0;
    for (int f0 = 0; f0 < nframes && ok; ++group) {
        const int g = std::min(G, nframes - f0);
        Slot &s = *slots_[static_cast<size_t>(group) % slots_.size()];
        finalize_slot(s);  // frees the slot (waits for the group that used it last)
        const bool direct = dst_pinned && !keep_unmapped;
        if (!src_pinned && !s.h_faces) CK(cudaMallocHost(&s.h_faces, slot_face_bytes_ * G));
        if (!direct && !s.h_out) CK(cudaMallocHost(&s.h_out, slot_out_bytes_ * G));
        // Only what the lens looks at is uploaded: plates with display != 0 (:764-766), and of
        // those only the texel rectangle the lensmap samples.  (TMA boxes may overhang the
        // rectangle; those texels are staged but never referenced by an entry.)
        cudaMemcpy3DBatchOp ops[BLINKY_MAX_PLATES * kMaxHostGroup];
        size_t nops = 0;
        for (int k = 0; k < g && ok; ++k) {
            const uint8_t *src = faces_host + static_cast<size_t>(f0 + k) * face_stride;
            uint8_t *d_frame = s.d_faces + static_cast<size_t>(k) * slot_face_bytes_;
            UploadRects ur;
            ur.n = 0;
            ur.first[0] = 0;
            ur.pitch = static_cast<uint32_t>(platesize_);
            const bool by_kernel = upload_by_kernel_ && platesize_ % 16 == 0 && reinterpret_cast<uintptr_t>(src) % 16 == 0 && face_stride % 16 == 0;
            for (int pl = 0; pl < numplates_; ++pl) {
                if (!display_[pl]) continue;
                const int *r = plate_rect_[pl];
                if (r[0] > r[2] || r[1] > r[3]) continue;
                if (by_kernel && src_pinned) {
                    const int xa = r[0] & ~15, xb = (r[2] + 16) & ~15;  // 16-byte columns covering [r0, r2]
                    ur.off[ur.n] = static_cast<uint32_t>(pl * ps2 + static_cast<size_t>(r[1]) * platesize_ + xa);
                    ur.vec_w[ur.n] = static_cast<uint32_t>((xb - xa) / 16);
                    ur.rows[ur.n] = static_cast<uint32_t>(r[3] - r[1] + 1);
                    ur.first[ur.n + 1] = ur.first[ur.n] + ur.vec_w[ur.n] * ur.rows[ur.n];
                    ++ur.n;
                    continue;
                }
                const size_t rw = static_cast<size_t>(r[2] - r[0] + 1), rh = static_cast<size_t>(r[3] - r[1] + 1);
                const size_t off = pl * ps2 + static_cast<size_t>(r[1]) * platesize_ + r[0];
                const uint8_t *from = src + off;
                if (!src_pinned) {
                    uint8_t *stage = s.h_faces + static_cast<size_t>(k) * slot_face_bytes_ + off;
                    for (size_t y = 0; y < rh; ++y) memcpy(stage + y * platesize_, from + y * platesize_, rw);
                    from = stage;
                }
                // a full-width rectangle is one contiguous run: copy it as such
                const bool contiguous = rw == static_cast<size_t>(platesize_);
                if (batch_copies_) {  // all rectangles of the group in ONE driver call (no gap between the DMA operations)
                    cudaMemcpy3DBatchOp &op = ops[nops++];
                    memset(&op, 0, sizeof op);
                    const size_t row = contiguous ? rw * rh : static_cast<size_t>(platesize_), rows = contiguous ? 1 : rh;
                    op.src.type = cudaMemcpyOperandTypePointer;
                    op.src.op.ptr.ptr = const_cast<uint8_t *>(from);
                    op.src.op.ptr.rowLength = row;
                    op.src.op.ptr.layerHeight = rows;
                    op.dst.type = cudaMemcpyOperandTypePointer;
                    op.dst.op.ptr.ptr = d_frame + off;
                    op.dst.op.ptr.rowLength = row;
                    op.dst.op.ptr.layerHeight = rows;
                    op.extent = make_cudaExtent(contiguous ? rw * rh : rw, rows, 1);
                    op.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
                    continue;
                }
                cudaError_t e = contiguous ? cudaMemcpyAsync(d_frame + off, from, rw * rh, cudaMemcpyHostToDevice, s.stream)
                                           : cudaMemcpy2DAsync(d_frame + off, static_cast<size_t>(platesize_), from, static_cast<size_t>(platesize_), rw, rh,
                                                               cudaMemcpyHostToDevice, s.stream);
                if (e != cudaSuccess) { ok = fail("cudaMemcpy2DAsync(H2D faces)", e); break; }
            }
            if (ok && ur.n > 0) {
                const uint32_t total = ur.first[ur.n];
                const unsigned blocks = std::min<unsigned>((total + 255) / 256, static_cast<unsigned>(sm_count_) * 8u);
                upload_rects_kernel<<<blocks, 256, 0, s.stream>>>(src, d_frame, ur);
                ++launches_;
            }
        }
        if (ok && nops > 0) {
            size_t fail_idx = 0;
            cudaError_t e = cudaMemcpy3DBatchAsync(nops, ops, &fail_idx, 0, s.stream);
            if (e != cudaSuccess) {
                // not available on this driver: fall back to one copy per rectangle, from now on
                cudaGetLastError();
                batch_copies_ = false;
                for (size_t k = 0; k < nops && ok; ++k) {
                    e = cudaMemcpy2DAsync(ops[k].dst.op.ptr.ptr, ops[k].dst.op.ptr.rowLength, ops[k].src.op.ptr.ptr, ops[k].src.op.ptr.rowLength,
                                          ops[k].extent.width, ops[k].extent.height, cudaMemcpyHostToDevice, s.stream);
                    if (e != cudaSuccess) ok = fail("cudaMemcpy2DAsync(H2D faces)", e);
                }
            }
        }
        if (!ok) break;
        s.dst = dst_host + static_cast<size_t>(f0) * dst_frame_stride;
        s.dst_frame_stride = dst_frame_stride;
        s.nf = g;
        // the warp kernel can store straight into the caller's pinned frames (posted PCIe writes, no
        // staging copy) when they are tightly packed
        const bool zero_copy_out = out_by_kernel_ && direct && dst_rowbytes == W && x0 == 0 && y0 == 0 &&
                                   reinterpret_cast<uintptr_t>(s.dst) % 16 == 0 && (g == 1 || dst_frame_stride % 16 == 0);
        if (!warp(s.d_faces, slot_face_bytes_, zero_copy_out ? s.dst : s.d_out, zero_copy_out ? dst_frame_stride : slot_out_bytes_, g, s.stream, false)) { ok = false; break; }
        s.dst_rowbytes = dst_rowbytes;
        s.x0 = x0;
        s.y0 = y0;
        s.keep_unmapped = keep_unmapped;
        s.direct = direct;
        cudaError_t e = cudaSuccess;
        const size_t frame = static_cast<size_t>(W) * H;
        if (zero_copy_out) {
        } else if (direct && dst_rowbytes == W && (g == 1 || (dst_frame_stride == frame && slot_out_bytes_ == frame))) {
            // tightly packed destination frames: the whole group is one contiguous run
            e = cudaMemcpyAsync(s.dst + static_cast<size_t>(y0) * dst_rowbytes + x0, s.d_out, frame * g, cudaMemcpyDeviceToHost, s.stream);
        } else if (direct) {
            for (int k = 0; k < g && e == cudaSuccess; ++k) {
                uint8_t *to = s.dst + static_cast<size_t>(k) * dst_frame_stride + static_cast<size_t>(y0) * dst_rowbytes + x0;
                const uint8_t *from = s.d_out + static_cast<size_t>(k) * slot_out_bytes_;
                e = dst_rowbytes == W ? cudaMemcpyAsync(to, from, frame, cudaMemcpyDeviceToHost, s.stream)
                                      : cudaMemcpy2DAsync(to, static_cast<size_t>(dst_rowbytes), from, static_cast<size_t>(W), static_cast<size_t>(W),
                                                          static_cast<size_t>(H), cudaMemcpyDeviceToHost, s.stream);
            }
        } else {
            e = cudaMemcpyAsync(s.h_out, s.d_out, slot_out_bytes_ * (g - 1) + frame, cudaMemcpyDeviceToHost, s.stream);
        }
        if (e != cudaSuccess) { ok = fail("cudaMemcpyAsync(D2H frame)", e); break; }
        e = cudaEventRecord(s.done, s.stream);
        if (e != cudaSuccess) { ok = fail("cudaEventRecord", e); break; }
        s.busy = true;
        f0 += g;
    }
    // drain in submission order
    for (size_t k = 0; k < slots_.size(); ++k) {
        Slot &s = *slots_[(static_cast<size_t>(group) + k) % slots_.size()];
        finalize_slot(s);
    }
    if (ok) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) ok = fail("warp_host", e);
    }
    return ok;
}

size_t WarpDevice::upload_bytes_per_frame() const {
    size_t n = 0;
    for (int pl = 0; pl < numplates_; ++pl) {
        const int *r = plate_rect_[pl];
        if (display_[pl] && r[0] <= r[2] && r[1] <= r[3]) n += static_cast<size_t>(r[2] - r[0] + 1) * static_cast<size_t>(r[3] - r[1] + 1);
    }
    return n;
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
