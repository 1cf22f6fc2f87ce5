#include "tile_plan.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "../../include/blinky_b200.h"
#include "parallel.h"

namespace blinky {

namespace {

struct RowPlan {
    std::vector<TileDesc> tiles;                  // in x order
    std::vector<std::vector<uint8_t>> blocks;     // entry block per tile (empty for EMPTY tiles)
    uint64_t box_bytes = 0, box_rows = 0;
    int stage_bytes = 0;
};

void plan_tile_row(const uint32_t *packed, int width, int height, int platesize, bool allow_box, int max_box_bytes, int h_gran, int tiles_x,
                   int ty, RowPlan &row) {
    const uint32_t ps = static_cast<uint32_t>(platesize);
    const uint32_t ps2 = ps * ps;
    std::vector<uint32_t> tile(kTilePixels);
    row.tiles.reserve(static_cast<size_t>(tiles_x));
    row.blocks.resize(static_cast<size_t>(tiles_x));
    for (int tx = 0; tx < tiles_x; ++tx) {
        const int x0 = tx * kTileW, y0 = ty * kTileH;
        // collect the tile (pixels beyond the frame edge are unmapped)
        bool any = false, one_plate = true, one_tint = true;
        int nvalid = 0;
        uint32_t plate = 0, tile_tint = BLINKY_LM_TINT_NONE;
        uint32_t minx = ~0u, miny = ~0u, maxx = 0, maxy = 0;
        for (int r = 0; r < kTileH; ++r) {
            for (int c = 0; c < kTileW; ++c) {
                uint32_t e = 0;
                if (y0 + r < height && x0 + c < width) e = packed[static_cast<size_t>(y0 + r) * width + x0 + c];
                tile[static_cast<size_t>(r) * kTileW + c] = e;
                if (!(e & BLINKY_LM_VALID)) continue;
                ++nvalid;
                const uint32_t idx = e & BLINKY_LM_INDEX_MASK;
                const uint32_t p = idx / ps2, rem = idx % ps2;
                const uint32_t py = rem / ps, px = rem % ps;
                if (!any) {
                    any = true;
                    plate = p;
                } else if (p != plate) {
                    one_plate = false;
                }
                const uint32_t tint = (e >> BLINKY_LM_TINT_SHIFT) & 7u;
                if (tint != BLINKY_LM_TINT_NONE) {
                    if (tile_tint == BLINKY_LM_TINT_NONE) tile_tint = tint;
                    else if (tint != tile_tint) one_tint = false;  // forward-built maps: the tint is sticky, the texel is the last writer's
                }
                minx = std::min(minx, px);
                maxx = std::max(maxx, px);
                miny = std::min(miny, py);
                maxy = std::max(maxy, py);
            }
        }
        TileDesc d;
        memset(&d, 0, sizeof d);
        d.px = static_cast<uint16_t>(x0);
        d.py = static_cast<uint16_t>(y0);
        if (!any) {
            d.type = TILE_EMPTY;
            row.tiles.push_back(d);
            continue;
        }
        bool box = allow_box && one_plate && one_tint;
        uint32_t bw = 0, bh = 0;
        // (TMA faults, "illegal instruction", unless the innermost coordinate is a multiple of 16 bytes:
        // scripts/tma_probe.cu)
        if (box) box = tile_box(minx, maxx, miny, maxy, h_gran, max_box_bytes, &minx, &bw, &bh);
        std::vector<uint8_t> &blk = row.blocks[static_cast<size_t>(tx)];
        if (box) {
            d.type = nvalid == kTilePixels ? TILE_BOX_FULL : TILE_BOX;
            d.plate = static_cast<uint8_t>(plate | (tile_tint << 3));
            d.box_x = static_cast<int16_t>(minx);
            d.box_y = static_cast<int16_t>(miny);
            d.box_w16 = static_cast<uint8_t>(bw / 16);
            d.box_h8 = static_cast<uint8_t>(bh / 8);
            blk.assign(kBoxBlockBytes, 0);
            uint16_t *ent = reinterpret_cast<uint16_t *>(blk.data());
            uint32_t *tinted = reinterpret_cast<uint32_t *>(blk.data() + kBoxEntryBytes);
            for (int lane = 0; lane < 32; ++lane) {
                for (int i = 0; i < 32; ++i) {
                    int r, c;
                    box_lane_pixel(lane, i, &r, &c);
                    bool tint;
                    ent[box_entry_slot(lane, i)] = box_entry(tile[static_cast<size_t>(r) * kTileW + c], ps, ps2, minx, miny, bw, &tint);
                    if (tint) tinted[lane] |= 1u << i;
                }
            }
            row.box_bytes += static_cast<uint64_t>(bw) * bh;
            row.box_rows += bh;
            row.stage_bytes = std::max(row.stage_bytes, static_cast<int>(bw * bh));
        } else {
            d.type = TILE_GATHER;
            blk.resize(kGatherBlockBytes);
            memcpy(blk.data(), tile.data(), kGatherBlockBytes);
        }
        row.tiles.push_back(d);
    }
}

}  // namespace

int plan_max_box_bytes(int max_box_bytes) {
    if (max_box_bytes <= 0) {
        max_box_bytes = kDefaultMaxBoxBytes;
        if (const char *e = getenv("BLINKY_MAX_BOX")) {
            const int v = atoi(e);
            if (v >= 128) max_box_bytes = v;
        }
    }
    return std::min(max_box_bytes, kBoxBytesLimit);
}

TilePlan make_tile_plan(const uint32_t *packed, int width, int height, int platesize, bool allow_box, int threads, int max_box_bytes) {
    TilePlan plan;
    max_box_bytes = plan_max_box_bytes(max_box_bytes);
    plan.max_box_bytes = max_box_bytes;
    plan.width = width;
    plan.height = height;
    plan.platesize = platesize;
    if (width > kMaxPlanExtent || height > kMaxPlanExtent) return plan;   // tile origins would not fit TileDesc::px / py
    plan.tiles_x = (width + kTileW - 1) / kTileW;
    plan.tiles_y = (height + kTileH - 1) / kTileH;
    // box heights come in multiples of 8 texel rows; if that needs more than kMaxShapes distinct
    // shapes (one TMA descriptor each), coarsen the heights and plan again
    std::vector<RowPlan> rows;
    for (int h_gran = 8;; h_gran *= 2) {
        rows.assign(static_cast<size_t>(plan.tiles_y), RowPlan());
        parallel_for(plan.tiles_y, threads, [&](int ty) {
            plan_tile_row(packed, width, height, platesize, allow_box, max_box_bytes, h_gran, plan.tiles_x, ty, rows[static_cast<size_t>(ty)]);
        });
        std::vector<uint16_t> shapes;
        for (const RowPlan &r : rows)
            for (const TileDesc &d : r.tiles)
                if (d.type == TILE_BOX || d.type == TILE_BOX_FULL) {
                    const uint16_t shape = static_cast<uint16_t>((d.box_w16 << 8) | d.box_h8);
                    if (std::find(shapes.begin(), shapes.end(), shape) == shapes.end()) shapes.push_back(shape);
                }
        plan.box_h_granularity = h_gran;
        if (static_cast<int>(shapes.size()) <= kMaxShapes) break;  // always true at 64 rows: 16 widths x 4 heights
    }
    // three passes in screen order: BOX tiles, GATHER tiles, EMPTY tiles
    size_t total = 0;
    for (const RowPlan &r : rows)
        for (const std::vector<uint8_t> &b : r.blocks) total += b.size();
    plan.entries.reserve(total + 16);
    plan.tiles.reserve(static_cast<size_t>(plan.tiles_x) * plan.tiles_y);
    for (int pass = 0; pass < 3; ++pass) {
        for (const RowPlan &r : rows) {
            for (size_t k = 0; k < r.tiles.size(); ++k) {
                TileDesc d = r.tiles[k];
                const bool is_box = d.type == TILE_BOX || d.type == TILE_BOX_FULL;
                const int cls = is_box ? 0 : d.type == TILE_GATHER ? 1 : 2;
                if (cls != pass) continue;
                d.entry_offset = static_cast<uint32_t>(plan.entries.size());
                plan.entries.insert(plan.entries.end(), r.blocks[k].begin(), r.blocks[k].end());
                plan.tiles.push_back(d);
                if (is_box) {
                    ++plan.n_box;
                    if (d.type == TILE_BOX_FULL) ++plan.n_box_full;
                    const uint16_t shape = static_cast<uint16_t>((d.box_w16 << 8) | d.box_h8);
                    size_t si = static_cast<size_t>(std::find(plan.shapes.begin(), plan.shapes.end(), shape) - plan.shapes.begin());
                    if (si == plan.shapes.size()) plan.shapes.push_back(shape);
                    plan.tiles.back().type = static_cast<uint8_t>(d.type | (si << kTileShapeShift));
                } else if (d.type == TILE_GATHER) {
                    ++plan.n_gather;
                } else {
                    ++plan.n_empty;
                }
            }
        }
    }
    plan.entries.resize(plan.entries.size() + 16);  // the kernels may prefetch one 16-byte vector past a block
    for (const RowPlan &r : rows) {
        plan.box_bytes += r.box_bytes;
        plan.box_rows += r.box_rows;
        plan.stage_bytes = std::max(plan.stage_bytes, r.stage_bytes);
    }
    plan.stage_bytes = (plan.stage_bytes + 127) / 128 * 128;
    return plan;
}

}  // namespace blinky
