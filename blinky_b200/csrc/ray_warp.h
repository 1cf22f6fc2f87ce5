// The warp from a ray field turned by a per-frame matrix (blinky_warp_device_rays, ray_warp.cu): what one launch
// needs, in host types, so that warp_device.cu can plan it without the kernel's translation unit.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>

#include "warp_device.h"

namespace blinky {

constexpr int kRayThreads = 256;   // threads per CTA of every ray-warp kernel

// The launch shape of a ray warp (ray_warp_shape, launch_plan.h): one thread per item — a 4-pixel quad of a row
// (quads) or one output pixel — in grid_x CTAs of kRayThreads per row of threads, and grid_y rows of
// frames_per_thread frames each.
struct RayWarpShape {
    bool quads;
    uint32_t nitems;            // items per frame: W * H / 4 quads or W * H pixels
    int frames_per_thread;
    uint32_t grid_x, grid_y;
};

// One ray warp as check_warp accepted it (r, q and what it derived in c), with what the launch adds.
struct RayWarpLaunch {
    const WarpRequest &r;
    const RayRequest &q;
    const CheckedWarp &c;       // view, pitch, layout (every plate of the globe, dense faces included) and pyramid levels
    const uint8_t *bg;          // background, [height][width], padded like a lensmap to whole quads
    const uint8_t *lut;         // [6][256] rubix tint LUTs
    const uint32_t *palette;    // RGBA: the palette table (tables: frame 0's)
    int width, height;
    RayWarpShape shape;
    bool rubix;
    const LensBuildParams &globe;   // FisheyeHost::device_params of the current globe at the view's size
    bool tables() const { return r.rgba && r.tables && r.table_stride != 0; }
};

// The name of the kernel a ray warp launches (last_kernel, and the failure it reports)
inline const char *ray_warp_kernel_name(RayFilter filter, int factor) {
    return filter == RayFilter::Trilinear ? "ray_trilinear_kernel"
           : filter == RayFilter::Bilinear ? "ray_bilinear_kernel"
           : factor > 1                    ? "ray_supersample_kernel"
                                           : "ray_warp_kernel";
}

// Launches the instance of L.q.filter's kernel in L.shape (for trilinear, one pyramid launch per level 1..lmax first).
// false with the CUDA error in *cuda_err; *name: the instance and launch shape of the warp kernel (last_kernel).
bool launch_ray_warp(const RayWarpLaunch &L, std::string *name, int *cuda_err);

}  // namespace blinky
