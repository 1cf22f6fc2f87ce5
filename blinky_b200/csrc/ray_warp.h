// The warp from a ray field turned by a per-frame matrix (blinky_warp_device_rays, ray_warp.cu): what one launch
// needs, in host types, so that warp_device.cu can plan it without the kernel's translation unit.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>

#include "face_layout.h"
#include "lens_device.h"
#include "ray_texel.h"   // kRayMaxLevels

namespace blinky {

constexpr int kRayThreads = 256;   // threads per CTA of every ray-warp kernel

// How each sample of a ray warp takes its colour: the nearest texel (ray_warp_kernel at factor 1,
// ray_supersample_kernel at 2-4), four texels blended (ray_bilinear_kernel, factor 1-4), or two mip levels' bilinear
// colours blended (the pyramid launches, then ray_trilinear_kernel, factor 1).  Every filter but Nearest at factor 1
// writes RGBA.
enum class RayFilter { Nearest, Bilinear, Trilinear };

// The launch shape of a ray warp (ray_warp_shape, launch_plan.h): one thread per item — a 4-pixel quad of a row
// (quads) or one output pixel — in grid_x CTAs of kRayThreads per row of threads, and grid_y rows of
// frames_per_thread frames each.
struct RayWarpShape {
    bool quads;
    uint32_t nitems;            // items per frame: W * H / 4 quads or W * H pixels
    int frames_per_thread;
    uint32_t grid_x, grid_y;
};

struct RayWarpLaunch {
    RayFilter filter;
    int factor;                 // k: k x k samples per pixel from a [k * height][k * width] field
    void *scratch;              // trilinear: frame 0's pyramid (16-byte aligned; frame f's at scratch + f * pyramid_bytes)
    size_t pyramid_bytes;       // trilinear: B, one frame's pyramid (ray_pyramid_levels)
    int lmax;                   // trilinear: the top level (0: no pyramid, plates of one texel)
    int level_size[kRayMaxLevels];        // trilinear: plate side of each level (ray_pyramid_levels)
    uint64_t level_off[kRayMaxLevels];    // trilinear: byte offset of each level L >= 1 in a frame's pyramid
    const float *rays;          // frame 0's field, float32[factor * height][factor * width][3]
    size_t ray_stride;          // bytes between frames' fields (0: one field for every frame)
    const float *xforms;        // frame 0's matrix, 9 floats row-major (nullptr: the rays as they are)
    size_t xform_stride;        // bytes between frames' matrices (0: one matrix for every frame)
    const void *faces;          // frame 0's faces, addressed through `layout`
    size_t face_stride;
    const uint8_t *bg;          // background, [height][width], padded like a lensmap to whole quads
    const uint8_t *lut;         // [6][256] rubix tint LUTs
    const uint32_t *palette;    // RGBA: the palette table (tables: frame 0's)
    size_t table_stride;        // tables: bytes between frames' tables
    void *out;                  // view origin of frame 0
    size_t out_stride;          // bytes between frames
    uint32_t pitch;             // bytes between output rows
    int width, height, nframes;
    RayWarpShape shape;
    bool rubix, rgba, keep, tables;
    LensBuildParams globe;      // FisheyeHost::device_params of the current globe at the view's size
    FaceLayoutParams layout;    // plate_base and rowbytes address every plate of the globe (dense faces included)
    void *stream;               // cudaStream_t
};

// The name of the kernel a ray warp launches (last_kernel, and the failure it reports)
inline const char *ray_warp_kernel_name(RayFilter filter, int factor) {
    return filter == RayFilter::Trilinear ? "ray_trilinear_kernel"
           : filter == RayFilter::Bilinear ? "ray_bilinear_kernel"
           : factor > 1                    ? "ray_supersample_kernel"
                                           : "ray_warp_kernel";
}

// Launches the instance of L.filter's kernel in L.shape (for trilinear, one pyramid launch per level 1..lmax first).
// false with the CUDA error in *cuda_err; *name: the instance and launch shape of the warp kernel (last_kernel).
bool launch_ray_warp(const RayWarpLaunch &L, std::string *name, int *cuda_err);

}  // namespace blinky
