// Tile plan: how the packed lensmap is re-laid out for the ring kernel (warp_device.cu).
//
// The screen is cut into 32x32-pixel tiles.  At lensmap-build time (host, once) each tile is
// classified:
//   EMPTY     no pixel of the tile is mapped -> background copy only
//   BOX       every mapped pixel reads one plate and the source texels fit a box of at most
//             `max_box_bytes` (<= 16 KB) -> the kernel stages that box in shared memory with one
//             TMA tensor load per frame and gathers from there; the tile's lensmap entries shrink
//             to 16 bits (offset inside the box, valid)
//   BOX_FULL  a BOX tile whose 1024 pixels are all mapped and inside the frame (no per-pixel
//             validity / background work)
//   GATHER    anything else (plate seams, singular points, very strong minification)
//             -> 32-bit entries, direct global gather
// Tiles are ordered BOX/BOX_FULL first, then GATHER, then EMPTY; entry blocks follow the same order
// and have fixed sizes, so a tile's block address is a function of its index alone.
//
// This replaces nothing in the reference (its lensmap is a flat array of pointers,
// the reference's engine/NQ/fisheye.c:427-430); it is the H100 data layout for the same information.
#pragma once

#include <cstdint>
#include <vector>

namespace blinky {

constexpr int kTileW = 32;
constexpr int kTileH = 32;
constexpr int kTilePixels = kTileW * kTileH;
constexpr int kBoxBytesLimit = 16384;      // 14-bit offsets
constexpr int kDefaultMaxBoxBytes = 8192;  // planner default (BLINKY_MAX_BOX overrides)
constexpr int kMaxBoxW = 256, kMaxBoxH = 256;  // TMA box dimensions are at most 256 elements
// A plan covers screens of at most 65536 x 65536 pixels: TileDesc::px / py hold tile origins in 16 bits.  For a
// wider or taller screen make_tile_plan returns a plan without tiles, and the flat kernels (K1 / K0, which address
// pixels by their dense index) serve the warp.
constexpr int kMaxPlanExtent = 65536;

enum TileType : uint8_t { TILE_EMPTY = 0, TILE_BOX = 1, TILE_GATHER = 2, TILE_BOX_FULL = 3 };
// A plan uses at most kMaxShapes distinct box shapes: the kernel receives one TMA descriptor per
// shape in its parameter block (no descriptor table in global memory, hence no tensormap-proxy
// fences).  TileDesc::type carries the shape index in its upper six bits.
constexpr int kMaxShapes = 64;
constexpr int kTileTypeMask = 3, kTileShapeShift = 2;

// 16-bit entry of a BOX tile
constexpr uint16_t kBoxValid = 0x8000;
constexpr uint16_t kBoxOffsetMask = 0x3FFF;
constexpr uint8_t kTileTintNone = 7;       // TileDesc tint of a BOX tile without tinted pixels

// Entry block of a BOX tile (kBoxBlockBytes):
//   [4][32][8] uint16 : load k (0..3) of lane l (0..31) is the 16 bytes at (k*32 + l)*16 -> fully
//                       coalesced 128-bit loads.  Entry j of load k is the lane's pixel i = 8k + j,
//                       which sits at tile row (l >> 3) + 4*(i >> 2), column 4*(l & 7) + (i & 3):
//                       a lane owns 8 quads (4 consecutive pixels each), a warp-level access covers
//                       4 tile rows.
//   [32] uint32       : bit i of word l = the lane's pixel i is tinted (rubix overlay).  All tinted pixels
//                       of a BOX tile share ONE tint (TileDesc::plate bits 3-5; in inverse-built maps it is
//                       the tile's plate, fisheye.c:1953-1958) — a tile with mixed tints is a GATHER tile —
//                       so the kernel applies one LUT row per tile and merges by byte masks.
constexpr int kBoxEntryBytes = kTilePixels * 2;
constexpr int kBoxTintBytes = 32 * 4;
constexpr int kBoxBlockBytes = kBoxEntryBytes + kBoxTintBytes;
// Entry block of a GATHER tile: [32][32] uint32 in the packed BLINKY_LM_* format, row-major.
constexpr int kGatherBlockBytes = kTilePixels * 4;

// The per-tile rules below are shared by make_tile_plan (host threads) and the device planner
// (tile_plan_device.cu), so that both produce the same plan byte for byte.
// (the same definition as face_layout.h's)
#if defined(__CUDACC__)
#define BLINKY_HD __host__ __device__ __forceinline__
#else
#define BLINKY_HD inline
#endif

BLINKY_HD void box_lane_pixel(int lane, int i, int *row, int *col) {
    *row = (lane >> 3) + 4 * (i >> 2);
    *col = 4 * (lane & 7) + (i & 3);
}

// Where entry i of lane `lane` sits among the [4][32][8] uint16 entries of a BOX block.
BLINKY_HD int box_entry_slot(int lane, int i) { return ((i >> 3) * 32 + lane) * 8 + (i & 7); }

// The box of a tile whose single-plate, single-tint mapped texels span [minx, maxx] x [miny, maxy]:
// origin x rounded down to 16 texels (TMA needs 16-byte aligned inner coordinates; the row coordinate is
// unconstrained), width a multiple of 16, height a multiple of h_gran.  False when the box is too large to
// stage, which makes the tile a GATHER tile.
BLINKY_HD bool tile_box(uint32_t minx, uint32_t maxx, uint32_t miny, uint32_t maxy, int h_gran, int max_box_bytes, uint32_t *box_x,
                     uint32_t *bw, uint32_t *bh) {
    const uint32_t g = static_cast<uint32_t>(h_gran);
    *box_x = minx & ~15u;
    *bw = ((maxx - *box_x + 1) + 15) / 16 * 16;
    *bh = ((maxy - miny + 1) + g - 1) / g * g;
    return !(*bw > static_cast<uint32_t>(kMaxBoxW) || *bh > static_cast<uint32_t>(kMaxBoxH) || *bw * *bh > static_cast<uint32_t>(max_box_bytes));
}

// 16-bit BOX entry of packed lensmap entry e in the box at (box_x, box_y), bw texels wide; unmapped pixels get
// offset 0 (a harmless read), not valid.  *tinted: the pixel carries a tint.
BLINKY_HD uint16_t box_entry(uint32_t e, uint32_t ps, uint32_t ps2, uint32_t box_x, uint32_t box_y, uint32_t bw, bool *tinted) {
    *tinted = false;
    if (!(e & 0x80000000u)) return 0;
    const uint32_t rem = (e & 0x0FFFFFFFu) % ps2;
    const uint32_t py = rem / ps, px = rem % ps;
    *tinted = ((e >> 28) & 7u) != 7u;
    return static_cast<uint16_t>(kBoxValid | ((py - box_y) * bw + (px - box_x)));
}

// Index of a box shape (w16 1..16, h8 1..32) in a 512-entry table.
BLINKY_HD int shape_slot(int w16, int h8) { return (w16 - 1) * 32 + (h8 - 1); }
constexpr int kShapeSlots = 16 * 32;

struct TileDesc {       // 16 bytes, read by the kernel
    uint32_t entry_offset;  // byte offset of the tile's entry block (= what the index-based rule gives)
    int16_t box_x, box_y;   // box origin in plate texel coordinates (may be < 0: TMA zero-fills)
    uint8_t plate;          // BOX tiles: plate (bits 0-2) | tint of the tile's tinted pixels << 3 (0-5, 7 = none tinted)
    uint8_t type;           // TileType | shape index << kTileShapeShift (BOX tiles)
    uint8_t box_w16;        // box width / 16  (1..16)
    uint8_t box_h8;         // box height / 8  (1..32)
    uint16_t px, py;        // tile origin on the screen, pixels
};
static_assert(sizeof(TileDesc) == 16, "TileDesc layout is part of the kernel ABI");

struct TilePlan {
    int width = 0, height = 0, platesize = 0;
    int tiles_x = 0, tiles_y = 0;
    int max_box_bytes = kDefaultMaxBoxBytes;   // planner cap used
    int stage_bytes = 0;                       // largest box of the plan, rounded up to 128
    std::vector<TileDesc> tiles;        // BOX / BOX_FULL tiles first (n_box of them), then GATHER, then EMPTY
    std::vector<uint8_t> entries;       // all entry blocks, tile-ordered
    std::vector<uint16_t> shapes;       // distinct (w16 << 8 | h8) used by BOX tiles, at most kMaxShapes; index = TileDesc shape index
    int box_h_granularity = 8;          // box heights are multiples of this (coarsened until the shapes fit)
    int n_empty = 0, n_box = 0, n_gather = 0, n_box_full = 0;  // n_box includes n_box_full
    uint64_t box_bytes = 0;             // sum of staged box sizes (bytes per frame through TMA)
    uint64_t box_rows = 0;              // sum of box heights (TMA requests per frame)
};

// packed: [height][width] entries in the BLINKY_LM_* format.  allow_box = false forces every
// non-empty tile to GATHER (e.g. platesize not a multiple of 16, which TMA cannot address).
// max_box_bytes <= 0: default / BLINKY_MAX_BOX.  Tile rows are classified on `threads` host
// threads; the result does not depend on the thread count.  A screen wider or taller than kMaxPlanExtent gets a
// plan without tiles.
TilePlan make_tile_plan(const uint32_t *packed, int width, int height, int platesize, bool allow_box, int threads = 1,
                        int max_box_bytes = 0);

// The box size cap a plan uses for a requested max_box_bytes (<= 0: the default, or BLINKY_MAX_BOX when set).
int plan_max_box_bytes(int max_box_bytes);

}  // namespace blinky
