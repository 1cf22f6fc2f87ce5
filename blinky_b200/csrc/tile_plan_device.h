// Tile planner for lensmaps that are already in device memory (blinky_set_lensmap_device): checks and normalises
// the map, derives what a build derives from it (FisheyeHost::finish_build) and writes the tile plan make_tile_plan
// would write, byte for byte, straight into the buffers the warps read.  Only the small results come back to the
// host.  CUDA types are kept out of this header.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "device_buffer.h"
#include "tile_plan.h"

namespace blinky {

// A map and its plan in device memory, owned until WarpDevice::install takes them over as its new generation.
struct DevicePlan {
    DeviceBuffer d_map;            // uint32_t[padded_pixels]: the normalised map (the padding unmapped)
    DeviceBuffer d_tiles;          // TileDesc[ntiles]
    DeviceBuffer d_entries;        // entry_bytes of entry blocks
    uint32_t ntiles = 0;
    size_t entry_bytes = 0;
    TilePlan plan;                 // sizes, counters, shapes and granularity (tiles / entries are not read)
    // what the host keeps (FisheyeHost::adopt_lensmap)
    int display[6] = {};
    int rect[6][4] = {};
    int64_t mapped = 0;
    std::vector<int32_t> span_off, spans;
};

// Plans the width x height map at d_packed (row pitch = width) on `stream` (a cudaStream_t) of CUDA device `device`,
// after the work already there, and returns once the results are complete.  BLINKY_OK, or BLINKY_E_INVALID for an
// entry whose index is beyond numplates * platesize^2 or whose tint is 6 (nothing is kept then), or BLINKY_E_CUDA;
// the reason in *why.  Sizes are checked by the caller (FisheyeHost::check_lensmap_size).
int plan_lensmap_device(int device, const uint32_t *d_packed, int width, int height, int platesize, int numplates, size_t padded_pixels,
                        void *stream, DevicePlan *out, std::string *why);

// Stages a map and the tile plan make_tile_plan made of it into *out on CUDA device `device`: the padded map with
// its padding unmapped, the tile table and the entry blocks.  BLINKY_OK, or BLINKY_E_CUDA with the reason in *why.
int stage_lensmap_host(int device, const uint32_t *packed, size_t npix, size_t padded_pixels, TilePlan plan, DevicePlan *out,
                       std::string *why);

}  // namespace blinky
