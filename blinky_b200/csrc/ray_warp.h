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

struct RayWarpLaunch {
    int factor;                 // 1: ray_warp_kernel; 2-4: ray_supersample_kernel, k x k samples per pixel (RGBA, never quads)
    bool bilinear;              // ray_bilinear_kernel, factor 1-4: k x k bilinear samples per pixel (RGBA, never quads)
    bool trilinear;             // the pyramid launches, then ray_trilinear_kernel (factor 1, RGBA, never quads)
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
    int frames_per_thread;      // ray_warp_frames_per_thread (launch_plan.h)
    bool quads;                 // ray_warp_quads (launch_plan.h)
    bool rubix, rgba, keep, tables;
    LensBuildParams globe;      // FisheyeHost::device_params of the current globe at the view's size
    FaceLayoutParams layout;    // plate_base and rowbytes address every plate of the globe (dense faces included)
    void *stream;               // cudaStream_t
};

// Launches ray_warp_kernel (factor 1), ray_supersample_kernel, ray_bilinear_kernel (bilinear) or, for trilinear, one
// pyramid launch per level 1..lmax and ray_trilinear_kernel for L.  false with the CUDA error in *cuda_err; *name: the
// instance and launch shape of the warp kernel (last_kernel).
bool launch_ray_warp(const RayWarpLaunch &L, std::string *name, int *cuda_err);

}  // namespace blinky
