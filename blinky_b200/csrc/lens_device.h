// Device-side lensmap construction (SURVEY section 8f rank 1): the reference evaluates the
// lens script once per screen pixel inside create_lensmap_inverse()
// (the reference's engine/NQ/fisheye.c:2084-2124, ~1 us .. 10 us per pixel through the Lua
// VM).  Here the script's lens_inverse is translated to CUDA C++ (lua_transpile.h),
// compiled for sm_90a with NVRTC at lens-load time, and evaluated for all W*H pixels by
// one kernel; the ray -> plate -> texel -> rubix tint tail of the pixel pipeline
// (fisheye.c:2023-2066, 1922-2013) runs in the same kernel with the host's exact float /
// double operation order.
//
// Forward-only lenses (SURVEY section 8f rank 3, fisheye.c:2126-2338) get the same treatment:
// lens_forward is evaluated at every plate grid point by a translated kernel, then static
// kernels in lens_device.cu replay the reference's stale-slot behaviour, rasterise the quads
// with the writer order encoded in atomicMax keys (last writer wins, tints stick) and resolve
// the map.
//
// Every pixel whose outcome is not provably identical to what the host's libm would give
// carries a risk bit and is re-evaluated by the host interpreter (fisheye_host.cpp), so the
// finished lensmap is the same as the all-host build.
//
// No CUDA types in this header.
#pragma once

#include <cstdint>
#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "device_buffer.h"

namespace blinky {

// Mirrors `struct LtParams` in the generated kernel source (lens_device.cu: kKernelSource).
struct LensBuildParams {
    int width, height, platesize, numplates;
    double scale;
    double rubix_block, rubix_pad, rubix_unit_px;
    double uv_dist[6];   // 0.5 / tan(fov/2) in double, per plate (ray_to_plate_uv)
    struct PlateF {
        float forward[3], right[3], up[3];
        float dist;
    } plates[6];
};

// candidate entry per pixel
constexpr uint32_t kCandValid = 0x80000000u;   // maps to a texel (bits 0..27 = texel index)
constexpr uint32_t kCandOnGrid = 0x40000000u;  // rubix padding: the pixel keeps its previous tint
constexpr uint32_t kCandRisk = 0x20000000u;    // not provably identical to the host result

// a grid point of the forward builder the host evaluated itself
struct ForwardPatch {
    uint32_t point;   // (plate * (ps+1) + j) * (ps+1) + i
    int32_t status;   // 1 = values, 0 = lens_forward returned nil
    int32_t lx, ly;
};

// the owner plane of the forward builder (globes with a globe_plate script): one byte per texel
// (plate * ps + py) * ps + px
constexpr uint8_t kOwnerOwned = 1u;  // globe_plate picks this texel's plate for the texel's ray
constexpr uint8_t kOwnerRisk = 2u;   // not provably the host's answer: the host decides
// a texel owner the host decided: the texel index, | kOwnerPatchOwned when the texel is owned
constexpr uint32_t kOwnerPatchOwned = 0x80000000u;

// a ray-map entry the host settled: pixel number (ly * width + lx) and packed lensmap entry
struct RayPatch {
    uint32_t pixel;
    uint32_t entry;
};

// an exported ray the host evaluated: pixel number (ly * width + lx) and the narrowed, unnormalised ray
struct RaySample {
    uint32_t pixel;
    float ray[3];
};

// True when a translated source defines lt_globe_plate (lua_transpile.h).
inline bool source_has_globe_plate(const std::string &lens_source) { return lens_source.find("\n#define LT_HAS_GLOBE_PLATE 1\n") != std::string::npos; }

// Builds lensmaps on the GPU for FisheyeHost; CPU-only contexts have none and take the interpreter.
class LensDevice {
public:
    explicit LensDevice(int device);
    ~LensDevice();

    // inverse lenses: one candidate entry per screen pixel into cand[width*height].
    // lens_source = transpile_prelude(true) + TranspileResult::source.  Returns false (reason in *err) when NVRTC is
    // unavailable, the source does not compile, or a CUDA call fails.
    bool build(const std::string &lens_source, const LensBuildParams &p, uint32_t *cand, std::string *err);
    // forward lenses, step 1: screen position of every plate grid point; `undecided` receives
    // the points the host has to evaluate itself.  When the source has a globe_plate, the texel
    // owners are computed too and `undecided_texels` receives the texels the host has to decide.
    bool forward_points(const std::string &lens_source, const LensBuildParams &p, std::vector<uint32_t> *undecided,
                        std::vector<uint32_t> *undecided_texels, std::string *err);
    // step 2: host results patched in (grid points, texel owners), quads rasterised in the reference's
    // order (last writer wins), map resolved.  messages: (order key, value) of every "%d > maxdiff" the
    // reference prints.
    bool forward_finish(const std::vector<ForwardPatch> &patches, const std::vector<uint32_t> &owner_patches, int32_t *idx, uint8_t *tint,
                        int display[6], std::vector<std::pair<uint32_t, int>> *messages, std::string *err);
    // step 2 for a ray export instead (DESIGN §3h): the same patches, stale slots and rasterised quads, then each
    // pixel's ray from its winning texel's quad (forward_raster.h: fwd_ray_pixel), normalised, the zero vector where no
    // texel draws, into d_rays (float32[height][width][3], device memory).  Everything runs on `stream` (a cudaStream_t)
    // after the work already there; returns once the field is written.  Nothing is printed or kept.
    bool forward_rays(const std::vector<ForwardPatch> &patches, const std::vector<uint32_t> &owner_patches, float *d_rays, void *stream,
                      std::string *err);
    // ray maps: the packed lensmap entry of each of the width * height float32 rays at d_rays (unnormalised, three per
    // pixel), on `stream` (a cudaStream_t) after the work already there, into a device map the builder keeps until its
    // next ray map (*d_map).  globe_source: the globe's globe_plate translated alone, or the bare prelude for argmax
    // globes.  Pixels whose plate decision is not provably the host's are written unmapped; *flagged receives them and
    // *flagged_rays their rays, for the host to settle.
    bool raymap(const std::string &globe_source, const LensBuildParams &p, const float *d_rays, void *stream, uint32_t **d_map,
                std::vector<uint32_t> *flagged, std::vector<float> *flagged_rays, std::string *err);
    // writes the settled entries into that map on `stream`; returns once they are there
    bool patch_entries(const std::vector<RayPatch> &patches, void *stream, std::string *err);
    // ray export: lens_inverse's ray at each of the p.width * p.height pixels of a build at p.scale, narrowed to float and
    // not normalised (zeros for nil), into d_rays (float32[height][width][3], device memory) on `stream` after the work
    // already there.  lens_source: the lens translated alone.  *flagged receives the pixels whose ray is not provably
    // the host's, for the host to evaluate; returns once the kernel has finished.
    bool rays(const std::string &lens_source, const LensBuildParams &p, float *d_rays, void *stream, std::vector<uint32_t> *flagged,
              std::string *err);
    // writes the host's rays into that field on `stream`; returns once they are there
    bool patch_rays(const std::vector<RaySample> &samples, float *d_rays, void *stream, std::string *err);
    // bytes from device memory on `stream`, after the work already there (a ray map that takes the host path)
    bool copy_to_host(void *dst, const void *d_src, size_t bytes, void *stream, std::string *err);
    // bytes to device memory on `stream`, after the work already there; returns once they are there (a ray export
    // that takes the host path)
    bool copy_to_device(void *d_dst, const void *src, size_t bytes, void *stream, std::string *err);
    // true while `stream` (a cudaStream_t) is capturing a graph, or when that cannot be asked
    static bool capturing(void *stream);

    // the fixed CUDA source appended to a translated lens (the per-pixel / per-grid-point tail);
    // exposed so that the CPU test-suite can run the very same text through a host shim.
    // globe_plate: the source defines lt_globe_plate — the inverse tail then lets it pick the plate and
    // the forward tail gains the owner kernel; without it the tails are unchanged.
    static std::string kernel_tail(bool forward, bool globe_plate = false);
    // the same for the ray-map kernel, appended to the globe's translated globe_plate (or the bare prelude)
    static std::string raymap_tail(bool globe_plate);
    // the same for the ray-export kernel, appended to the lens translated alone
    static std::string rays_tail();
    // the math probe kernel (blinky_probe_math), appended to the bare prelude
    static std::string probe_tail();

    // test hook: one prelude wrapper or IEEE operation (BLINKY_PROBE_*) on n exact arguments in device memory, value
    // and bound into d_v and d_e, on `stream` after the work already there; returns once they are written.
    // prelude: transpile_prelude(true), the text every lens unit starts with.
    bool probe_math(const std::string &prelude, int op, const double *d_a, const double *d_b, double *d_v, double *d_e, size_t n,
                    void *stream, std::string *err);

    // compile only (no GPU needed): used by the CPU test-suite and by build()
    static bool compile(const std::string &lens_source, bool forward, std::vector<char> *cubin, std::string *log);
    // a complete unit, with the NVRTC options of every lens unit (no GPU needed)
    static bool compile_unit(const std::string &src, std::vector<char> *cubin, std::string *log);

    double last_compile_ms() const { return compile_ms_; }
    double last_kernel_ms() const { return kernel_ms_; }
    double last_ray_kernel_ms() const { return ray_kernel_ms_; }  // forward_rays: fwd_ray_kernel alone

private:
    struct Module;
    struct ForwardState;
    enum Unit { kInverseUnit, kForwardUnit, kRaymapUnit, kRaysUnit, kProbeUnit };
    Module *module_for(const std::string &source, Unit unit, std::string *err);
    // forward steps 2-3 on `stream`: the host's grid points and texel owners patched in, then (raster_forward) the
    // stale slots replayed and every texel's quad rasterised into f.keys
    bool patch_forward(ForwardState &f, const std::vector<ForwardPatch> &patches, const std::vector<uint32_t> &owner_patches, void *stream,
                       std::string *err);
    void raster_forward(ForwardState &f, void *stream);
    int device_;
    std::map<std::string, std::unique_ptr<Module>> cache_;  // by unit + source text
    std::unique_ptr<ForwardState> fwd_;  // between forward_points() and forward_finish()
    DeviceBuffer ray_flagged_;  // ray maps and exports: [0] the flagged count, then the flagged pixels
    DeviceBuffer ray_map_;      // ray maps: the last map, ray_map_pixels_ entries
    size_t ray_map_pixels_ = 0;
    double compile_ms_ = 0, kernel_ms_ = 0, ray_kernel_ms_ = 0;
};

}  // namespace blinky
