// The tile planner on the GPU (tile_plan_device.h).  Passes, all on the caller's stream:
//   1. per pixel (one CTA per row): check and normalise the entries, and reduce the display flags, per-plate
//      texel rectangles, the mapped count and the number of mapped runs of each row;
//   2. per tile (one warp per tile): plate and tint uniformity and texel bounds, the tile's class and box
//      (tile_box, shared with make_tile_plan), and the first BOX tile of each box shape (atomicMin in a
//      512-entry table); repeated with coarser box heights while the shapes do not fit kMaxShapes;
//   3. exclusive scans (CUB) of the tile classes and of the runs per row;
//   4. per tile: the descriptor and entry block at the tile's slot (box_entry, shared with make_tile_plan);
//   5. per row (one warp per row): the row spans.
// The host waits twice: for the counts and shapes after pass 2, and for the spans at the end.
#include "tile_plan_device.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>
#include <cub/device/device_scan.cuh>

#include "../../include/blinky_b200.h"

namespace blinky {

namespace {

constexpr int kMaxPlanPlates = 6;
constexpr int kRowThreads = 256;
constexpr int kTilesPerCta = 8;  // one warp each

struct MapSummary {
    unsigned long long mapped;
    unsigned long long runs;     // mapped runs over all rows (row spans)
    unsigned long long bad_at;   // smallest pixel index of a refused entry (~0: none)
    int rect[kMaxPlanPlates][4];
};

struct TileSummary {
    unsigned n_box, n_gather, n_box_full;
    int stage_bytes;
    unsigned long long box_bytes, box_rows;
    int shape_first[kShapeSlots];  // first BOX tile (screen order) of each shape; INT_MAX: unused
};

__global__ void check_map_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, int width, uint32_t ps, uint32_t limit,
                                 MapSummary *sum, int32_t *row_runs) {
    __shared__ int rect[kMaxPlanPlates][4];
    __shared__ unsigned mapped, runs;
    const int y = blockIdx.x;
    if (threadIdx.x < kMaxPlanPlates * 4) rect[threadIdx.x / 4][threadIdx.x % 4] = threadIdx.x % 4 < 2 ? static_cast<int>(ps) : -1;
    if (threadIdx.x == 0) mapped = runs = 0;
    __syncthreads();
    const uint32_t ps2 = ps * ps;
    const size_t row = static_cast<size_t>(y) * static_cast<size_t>(width);
    unsigned my_mapped = 0, my_runs = 0;
    for (int x = threadIdx.x; x < width; x += blockDim.x) {
        const uint32_t e = in[row + x];
        if (!(e & BLINKY_LM_VALID)) {
            out[row + x] = BLINKY_LM_TINT_NONE << BLINKY_LM_TINT_SHIFT;
            continue;
        }
        out[row + x] = e;
        const uint32_t idx = e & BLINKY_LM_INDEX_MASK;
        if (idx >= limit || ((e >> BLINKY_LM_TINT_SHIFT) & 7u) == 6u) {
            atomicMin(&sum->bad_at, static_cast<unsigned long long>(row + x));
            continue;
        }
        ++my_mapped;
        if (x == 0 || !(in[row + x - 1] & BLINKY_LM_VALID)) ++my_runs;
        const uint32_t plate = idx / ps2, rem = idx % ps2;
        const int ty = static_cast<int>(rem / ps), tx = static_cast<int>(rem % ps);
        atomicMin(&rect[plate][0], tx);
        atomicMin(&rect[plate][1], ty);
        atomicMax(&rect[plate][2], tx);
        atomicMax(&rect[plate][3], ty);
    }
    if (my_mapped) atomicAdd(&mapped, my_mapped);
    if (my_runs) atomicAdd(&runs, my_runs);
    __syncthreads();
    if (threadIdx.x < kMaxPlanPlates * 4) {
        const int p = threadIdx.x / 4, k = threadIdx.x % 4, v = rect[p][k];
        if (rect[p][0] <= rect[p][2]) {
            if (k < 2) atomicMin(&sum->rect[p][k], v);
            else atomicMax(&sum->rect[p][k], v);
        }
    }
    if (threadIdx.x == 0) {
        row_runs[y] = static_cast<int32_t>(runs);
        if (mapped) atomicAdd(&sum->mapped, static_cast<unsigned long long>(mapped));
        if (runs) atomicAdd(&sum->runs, static_cast<unsigned long long>(runs));
    }
}

struct PlanGeometry {
    int width, height, tiles_x;
    uint32_t ntiles, ps, ps2;
    bool allow_box;
    int h_gran, max_box_bytes;
};

// the 32 entries of column `lane` of a tile, row r in e[r] (0 beyond the frame, like make_tile_plan)
__device__ __forceinline__ uint32_t tile_entry(const uint32_t *map, const PlanGeometry &g, int x0, int y0, int r, int c) {
    const int x = x0 + c, y = y0 + r;
    return x < g.width && y < g.height ? map[static_cast<size_t>(y) * g.width + x] : 0u;
}

// screen-order descriptor of every tile (entry_offset and shape index still 0) and its class in the scan input:
// 1 for BOX / BOX_FULL, 1 << 32 for GATHER, 0 for EMPTY
__global__ void classify_kernel(const uint32_t *__restrict__ map, PlanGeometry g, TileDesc *desc, unsigned long long *cls, TileSummary *sum) {
    const uint32_t t = blockIdx.x * kTilesPerCta + threadIdx.x / 32;
    const int lane = threadIdx.x % 32;
    if (t >= g.ntiles) return;
    const int x0 = static_cast<int>(t % g.tiles_x) * kTileW, y0 = static_cast<int>(t / g.tiles_x) * kTileH;
    unsigned nvalid = 0, pmin = ~0u, pmax = 0, tmin = 7, tmax = 0, minx = ~0u, maxx = 0, miny = ~0u, maxy = 0;
    for (int r = 0; r < kTileH; ++r) {
        const uint32_t e = tile_entry(map, g, x0, y0, r, lane);
        if (!(e & BLINKY_LM_VALID)) continue;
        ++nvalid;
        const uint32_t idx = e & BLINKY_LM_INDEX_MASK, p = idx / g.ps2, rem = idx % g.ps2, py = rem / g.ps, px = rem % g.ps;
        const uint32_t tint = (e >> BLINKY_LM_TINT_SHIFT) & 7u;
        pmin = min(pmin, p), pmax = max(pmax, p);
        if (tint != BLINKY_LM_TINT_NONE) tmin = min(tmin, tint), tmax = max(tmax, tint);
        minx = min(minx, px), maxx = max(maxx, px), miny = min(miny, py), maxy = max(maxy, py);
    }
    const unsigned full = 0xffffffffu;
    nvalid = __reduce_add_sync(full, nvalid);
    pmin = __reduce_min_sync(full, pmin), pmax = __reduce_max_sync(full, pmax);
    tmin = __reduce_min_sync(full, tmin), tmax = __reduce_max_sync(full, tmax);
    minx = __reduce_min_sync(full, minx), maxx = __reduce_max_sync(full, maxx);
    miny = __reduce_min_sync(full, miny), maxy = __reduce_max_sync(full, maxy);
    if (lane != 0) return;
    TileDesc d = {};
    d.px = static_cast<uint16_t>(x0);
    d.py = static_cast<uint16_t>(y0);
    unsigned long long c = 0;
    if (nvalid == 0) {
        d.type = TILE_EMPTY;
    } else {
        // tinted pixels share one tint when their smallest and largest tints agree (tmin 7: none is tinted)
        bool box = g.allow_box && pmin == pmax && (tmin == BLINKY_LM_TINT_NONE || tmin == tmax);
        uint32_t bx = 0, bw = 0, bh = 0;
        if (box) box = tile_box(minx, maxx, miny, maxy, g.h_gran, g.max_box_bytes, &bx, &bw, &bh);
        if (box) {
            d.type = nvalid == kTilePixels ? TILE_BOX_FULL : TILE_BOX;
            d.plate = static_cast<uint8_t>(pmin | (tmin << 3));
            d.box_x = static_cast<int16_t>(bx);
            d.box_y = static_cast<int16_t>(miny);
            d.box_w16 = static_cast<uint8_t>(bw / 16);
            d.box_h8 = static_cast<uint8_t>(bh / 8);
            c = 1;
            atomicAdd(&sum->n_box, 1u);
            if (d.type == TILE_BOX_FULL) atomicAdd(&sum->n_box_full, 1u);
            atomicAdd(&sum->box_bytes, static_cast<unsigned long long>(bw * bh));
            atomicAdd(&sum->box_rows, static_cast<unsigned long long>(bh));
            atomicMax(&sum->stage_bytes, static_cast<int>(bw * bh));
            atomicMin(&sum->shape_first[shape_slot(d.box_w16, d.box_h8)], static_cast<int>(t));
        } else {
            d.type = TILE_GATHER;
            c = 1ull << 32;
            atomicAdd(&sum->n_gather, 1u);
        }
    }
    desc[t] = d;
    cls[t] = c;
}

// every tile's descriptor and entry block at its slot: BOX tiles, then GATHER, then EMPTY, each in screen order
__global__ void write_plan_kernel(const uint32_t *__restrict__ map, PlanGeometry g, const TileDesc *__restrict__ desc,
                                  const unsigned long long *__restrict__ before, const uint8_t *__restrict__ shape_index, uint32_t n_box,
                                  uint32_t n_gather, TileDesc *tiles, uint8_t *entries) {
    const uint32_t t = blockIdx.x * kTilesPerCta + threadIdx.x / 32;
    const int lane = threadIdx.x % 32;
    if (t >= g.ntiles) return;
    TileDesc d = desc[t];
    const uint32_t box_before = static_cast<uint32_t>(before[t]), gather_before = static_cast<uint32_t>(before[t] >> 32);
    const int type = d.type;
    const bool is_box = type == TILE_BOX || type == TILE_BOX_FULL;
    uint32_t slot;
    uint64_t off;
    if (is_box) {
        slot = box_before;
        off = static_cast<uint64_t>(slot) * kBoxBlockBytes;
    } else if (type == TILE_GATHER) {
        slot = n_box + gather_before;
        off = static_cast<uint64_t>(n_box) * kBoxBlockBytes + static_cast<uint64_t>(gather_before) * kGatherBlockBytes;
    } else {
        slot = n_box + n_gather + (t - box_before - gather_before);
        off = static_cast<uint64_t>(n_box) * kBoxBlockBytes + static_cast<uint64_t>(n_gather) * kGatherBlockBytes;
    }
    const int x0 = d.px, y0 = d.py;
    if (is_box) {
        const uint32_t bx = static_cast<uint32_t>(d.box_x), by = static_cast<uint32_t>(d.box_y), bw = d.box_w16 * 16u;
        uint32_t tinted = 0;
        for (int k = 0; k < 4; ++k) {
            uint16_t v[8];
            for (int j = 0; j < 8; ++j) {
                const int i = 8 * k + j;
                int r, c;
                box_lane_pixel(lane, i, &r, &c);
                bool tint;
                v[j] = box_entry(tile_entry(map, g, x0, y0, r, c), g.ps, g.ps2, bx, by, bw, &tint);
                if (tint) tinted |= 1u << i;
            }
            uint4 q;
            q.x = v[0] | static_cast<uint32_t>(v[1]) << 16;
            q.y = v[2] | static_cast<uint32_t>(v[3]) << 16;
            q.z = v[4] | static_cast<uint32_t>(v[5]) << 16;
            q.w = v[6] | static_cast<uint32_t>(v[7]) << 16;
            *reinterpret_cast<uint4 *>(entries + off + box_entry_slot(lane, 8 * k) * 2) = q;
        }
        reinterpret_cast<uint32_t *>(entries + off + kBoxEntryBytes)[lane] = tinted;
        d.type = static_cast<uint8_t>(type | (shape_index[shape_slot(d.box_w16, d.box_h8)] << kTileShapeShift));
    } else if (type == TILE_GATHER) {
        uint32_t *blk = reinterpret_cast<uint32_t *>(entries + off);
        for (int r = 0; r < kTileH; ++r) blk[r * kTileW + lane] = tile_entry(map, g, x0, y0, r, lane);
    }
    if (lane == 0) {
        d.entry_offset = static_cast<uint32_t>(off);
        tiles[slot] = d;
    }
}

// the [x0, x1) runs of mapped pixels of each row (one warp per row), pairs from spans[2 * span_off[y]]
__global__ void row_spans_kernel(const uint32_t *__restrict__ map, int width, int height, const int32_t *__restrict__ span_off, int32_t *spans) {
    const int y = blockIdx.x * kTilesPerCta + threadIdx.x / 32;
    const int lane = threadIdx.x % 32;
    if (y >= height) return;
    const uint32_t *row = map + static_cast<size_t>(y) * width;
    int32_t *out = spans + 2 * static_cast<size_t>(span_off[y]);
    const unsigned below = (1u << lane) - 1u;
    int nstart = 0, nend = 0;
    bool prev = false;
    for (int x0 = 0; x0 < width; x0 += 32) {
        const int x = x0 + lane;
        const unsigned v = __ballot_sync(0xffffffffu, x < width && (row[x] & BLINKY_LM_VALID));
        const unsigned p = (v << 1) | (prev ? 1u : 0u);  // bit l: pixel x - 1 is mapped
        const unsigned starts = v & ~p, ends = ~v & p;
        if ((starts >> lane) & 1u) out[2 * (nstart + __popc(starts & below))] = x;
        if ((ends >> lane) & 1u) out[2 * (nend + __popc(ends & below)) + 1] = x;
        nstart += __popc(starts);
        nend += __popc(ends);
        prev = (v >> 31) & 1u;
    }
    if (prev && lane == 0) out[2 * nend + 1] = width;  // a run that reaches the last column
}

// *why = "<who>: <call>: <CUDA error>"
int cuda_failed(std::string *why, const char *who, const char *what, cudaError_t e) {
    char buf[256];
    snprintf(buf, sizeof buf, "%s: %s: %s", who, what, cudaGetErrorString(e));
    *why = buf;
    return BLINKY_E_CUDA;
}

}  // namespace

// (on the way out, every buffer is freed by its owner: the temporaries here, *out's by the caller's DevicePlan)
#define PK(call)                                                           \
    do {                                                                   \
        const cudaError_t e_ = static_cast<cudaError_t>(call);             \
        if (e_ != cudaSuccess) return cuda_failed(why, who, #call, e_); \
    } while (0)

int plan_lensmap_device(int device, const uint32_t *d_packed, int width, int height, int platesize, int numplates, size_t padded_pixels,
                        void *stream, DevicePlan *out, std::string *why) {
    const char *who = "blinky_set_lensmap_device";
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t npix = static_cast<size_t>(width) * height;
    const uint32_t ps = static_cast<uint32_t>(platesize), ps2 = ps * ps;
    *out = DevicePlan();
    TilePlan &plan = out->plan;
    plan.width = width;
    plan.height = height;
    plan.platesize = platesize;
    plan.max_box_bytes = plan_max_box_bytes(0);
    const bool tiled = width <= kMaxPlanExtent && height <= kMaxPlanExtent;  // (see make_tile_plan)
    if (tiled) {
        plan.tiles_x = (width + kTileW - 1) / kTileW;
        plan.tiles_y = (height + kTileH - 1) / kTileH;
    }
    const uint32_t ntiles = static_cast<uint32_t>(plan.tiles_x) * static_cast<uint32_t>(plan.tiles_y);
    DeviceBuffer msum_buf, tsum_buf, row_runs_buf, span_off_buf, spans_buf, desc_buf, cls_buf, before_buf, shape_index_buf, scratch;

    // 1. per pixel
    PK(cudaSetDevice(device));
    PK(out->d_map.alloc(padded_pixels * sizeof(uint32_t)));
    PK(msum_buf.alloc(sizeof(MapSummary)));
    PK(row_runs_buf.alloc((static_cast<size_t>(height) + 1) * sizeof(int32_t)));
    PK(span_off_buf.alloc((static_cast<size_t>(height) + 1) * sizeof(int32_t)));
    uint32_t *d_map = out->d_map.as<uint32_t>();
    MapSummary *d_msum = msum_buf.as<MapSummary>();
    int32_t *d_row_runs = row_runs_buf.as<int32_t>(), *d_span_off = span_off_buf.as<int32_t>();
    MapSummary msum_init = {0, 0, ~0ull, {}};
    for (int p = 0; p < kMaxPlanPlates; ++p) {
        msum_init.rect[p][0] = msum_init.rect[p][1] = platesize;
        msum_init.rect[p][2] = msum_init.rect[p][3] = -1;
    }
    PK(cudaMemcpyAsync(d_msum, &msum_init, sizeof msum_init, cudaMemcpyHostToDevice, s));
    if (padded_pixels > npix) PK(cudaMemsetAsync(d_map + npix, 0, (padded_pixels - npix) * sizeof(uint32_t), s));
    PK(cudaMemsetAsync(d_row_runs + height, 0, sizeof(int32_t), s));
    const uint32_t limit = static_cast<uint32_t>(static_cast<uint64_t>(ps2) * static_cast<uint32_t>(numplates));
    check_map_kernel<<<height, kRowThreads, 0, s>>>(d_packed, d_map, width, ps, limit, d_msum, d_row_runs);
    PK(cudaGetLastError());

    // 2. per tile, at box heights in multiples of 8 rows, coarsened until the shapes fit
    PlanGeometry g = {width, height, plan.tiles_x, ntiles, ps, ps2, platesize % 16 == 0, 8, plan.max_box_bytes};
    const unsigned tile_ctas = (ntiles + kTilesPerCta - 1) / kTilesPerCta;
    TileSummary tsum = {};
    if (ntiles) {
        PK(tsum_buf.alloc(sizeof(TileSummary)));
        PK(desc_buf.alloc(ntiles * sizeof(TileDesc)));
        PK(cls_buf.alloc(ntiles * sizeof(unsigned long long)));
        PK(before_buf.alloc(ntiles * sizeof(unsigned long long)));
    }
    TileSummary *d_tsum = tsum_buf.as<TileSummary>();
    TileDesc *d_desc = desc_buf.as<TileDesc>();
    unsigned long long *d_cls = cls_buf.as<unsigned long long>(), *d_before = before_buf.as<unsigned long long>();
    auto classify = [&]() -> cudaError_t {
        memset(&tsum, 0, sizeof tsum);
        std::fill(tsum.shape_first, tsum.shape_first + kShapeSlots, INT_MAX);
        cudaError_t e = cudaMemcpyAsync(d_tsum, &tsum, sizeof tsum, cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return e;
        classify_kernel<<<tile_ctas, kTilesPerCta * 32, 0, s>>>(d_map, g, d_desc, d_cls, d_tsum);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(&tsum, d_tsum, sizeof tsum, cudaMemcpyDeviceToHost, s);
        return e;
    };
    if (ntiles) PK(classify());
    MapSummary msum;
    PK(cudaMemcpyAsync(&msum, d_msum, sizeof msum, cudaMemcpyDeviceToHost, s));
    PK(cudaStreamSynchronize(s));
    if (msum.bad_at != ~0ull) {
        uint32_t e = 0;
        cudaMemcpy(&e, d_packed + msum.bad_at, sizeof e, cudaMemcpyDeviceToHost);
        char buf[200];
        snprintf(buf, sizeof buf, "blinky_set_lensmap_device: entry 0x%08x at (%llu, %llu): %s", e, msum.bad_at % static_cast<unsigned>(width),
                 msum.bad_at / static_cast<unsigned>(width), ((e >> 28) & 7u) == 6u ? "tint 6 is not a tint" : "texel index beyond numplates * platesize^2");
        *why = buf;
        return BLINKY_E_INVALID;
    }
    std::vector<std::pair<int, uint16_t>> first;  // (first BOX tile, shape)
    for (;;) {
        first.clear();
        if (ntiles)
            for (int w16 = 1; w16 <= 16; ++w16)
                for (int h8 = 1; h8 <= 32; ++h8) {
                    const int f = tsum.shape_first[shape_slot(w16, h8)];
                    if (f != INT_MAX) first.push_back({f, static_cast<uint16_t>((w16 << 8) | h8)});
                }
        plan.box_h_granularity = g.h_gran;
        if (static_cast<int>(first.size()) <= kMaxShapes) break;  // always true at 64 rows: 16 widths x 4 heights
        g.h_gran *= 2;
        PK(classify());
        PK(cudaStreamSynchronize(s));
    }
    std::sort(first.begin(), first.end());
    uint8_t shape_index[kShapeSlots] = {};
    for (size_t i = 0; i < first.size(); ++i) {
        plan.shapes.push_back(first[i].second);
        shape_index[shape_slot(first[i].second >> 8, first[i].second & 0xff)] = static_cast<uint8_t>(i);
    }
    plan.n_box = static_cast<int>(tsum.n_box);
    plan.n_gather = static_cast<int>(tsum.n_gather);
    plan.n_box_full = static_cast<int>(tsum.n_box_full);
    plan.n_empty = static_cast<int>(ntiles) - plan.n_box - plan.n_gather;
    plan.box_bytes = tsum.box_bytes;
    plan.box_rows = tsum.box_rows;
    plan.stage_bytes = (tsum.stage_bytes + 127) / 128 * 128;

    // 3. scans: tile slots (BOX and GATHER tiles before each tile) and span offsets
    size_t scratch_bytes = 0, b = 0;
    PK(cub::DeviceScan::ExclusiveSum(nullptr, b, d_row_runs, d_span_off, height + 1, s));
    scratch_bytes = b;
    if (ntiles) {
        PK(cub::DeviceScan::ExclusiveSum(nullptr, b, d_cls, d_before, ntiles, s));
        scratch_bytes = std::max(scratch_bytes, b);
    }
    PK(scratch.alloc(scratch_bytes));
    PK(cub::DeviceScan::ExclusiveSum(scratch.get(), scratch_bytes, d_row_runs, d_span_off, height + 1, s));

    // 4. descriptors and entry blocks
    if (ntiles) {
        PK(cub::DeviceScan::ExclusiveSum(scratch.get(), scratch_bytes, d_cls, d_before, ntiles, s));
        out->ntiles = ntiles;
        out->entry_bytes = static_cast<size_t>(plan.n_box) * kBoxBlockBytes + static_cast<size_t>(plan.n_gather) * kGatherBlockBytes + 16;
        PK(out->d_tiles.alloc(ntiles * sizeof(TileDesc)));
        PK(out->d_entries.alloc(out->entry_bytes));
        PK(shape_index_buf.alloc(sizeof shape_index));
        PK(cudaMemcpyAsync(shape_index_buf.get(), shape_index, sizeof shape_index, cudaMemcpyHostToDevice, s));
        PK(cudaMemsetAsync(out->d_entries.as<uint8_t>() + out->entry_bytes - 16, 0, 16, s));  // the kernels may prefetch one 16-byte vector past a block
        write_plan_kernel<<<tile_ctas, kTilesPerCta * 32, 0, s>>>(d_map, g, d_desc, d_before, shape_index_buf.as<uint8_t>(), tsum.n_box, tsum.n_gather,
                                                                 out->d_tiles.as<TileDesc>(), out->d_entries.as<uint8_t>());
        PK(cudaGetLastError());
    }

    // 5. row spans
    if (msum.runs) {
        PK(spans_buf.alloc(msum.runs * 2 * sizeof(int32_t)));
        row_spans_kernel<<<(height + kTilesPerCta - 1) / kTilesPerCta, kTilesPerCta * 32, 0, s>>>(d_map, width, height, d_span_off, spans_buf.as<int32_t>());
        PK(cudaGetLastError());
    }
    out->span_off.resize(static_cast<size_t>(height) + 1);
    out->spans.resize(msum.runs * 2);
    PK(cudaMemcpyAsync(out->span_off.data(), d_span_off, out->span_off.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (msum.runs) PK(cudaMemcpyAsync(out->spans.data(), spans_buf.get(), out->spans.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PK(cudaStreamSynchronize(s));
    out->mapped = static_cast<int64_t>(msum.mapped);
    for (int p = 0; p < kMaxPlanPlates; ++p) {
        for (int k = 0; k < 4; ++k) out->rect[p][k] = msum.rect[p][k];
        out->display[p] = msum.rect[p][0] <= msum.rect[p][2] ? 1 : 0;  // a plate is displayed when some mapped pixel samples it
    }
    return BLINKY_OK;
}

int stage_lensmap_host(int device, const uint32_t *packed, size_t npix, size_t padded_pixels, TilePlan plan, DevicePlan *out,
                       std::string *why) {
    const char *who = "lensmap upload";
    *out = DevicePlan();
    PK(cudaSetDevice(device));
    PK(out->d_map.alloc(padded_pixels * sizeof(uint32_t)));
    PK(cudaMemset(out->d_map.as<uint32_t>() + npix, 0, (padded_pixels - npix) * sizeof(uint32_t)));  // padding entries are unmapped
    PK(cudaMemcpy(out->d_map.get(), packed, npix * sizeof(uint32_t), cudaMemcpyHostToDevice));
    if (!plan.tiles.empty()) {
        out->ntiles = static_cast<uint32_t>(plan.tiles.size());
        out->entry_bytes = plan.entries.size();
        PK(out->d_tiles.alloc(plan.tiles.size() * sizeof(TileDesc)));
        PK(cudaMemcpy(out->d_tiles.get(), plan.tiles.data(), plan.tiles.size() * sizeof(TileDesc), cudaMemcpyHostToDevice));
        PK(out->d_entries.alloc(plan.entries.size()));
        PK(cudaMemcpy(out->d_entries.get(), plan.entries.data(), plan.entries.size(), cudaMemcpyHostToDevice));
    }
    out->plan = std::move(plan);
    return BLINKY_OK;
}
#undef PK

}  // namespace blinky
