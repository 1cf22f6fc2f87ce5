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
#include <string>
#include <utility>
#include <vector>

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

// What FisheyeHost needs from a GPU (implemented by LensDevice).  CPU-only contexts have no
// builder and take the interpreter.
class DeviceLensBuilder {
public:
    virtual ~DeviceLensBuilder() {}
    // inverse lenses: one candidate entry per screen pixel
    virtual bool build(const std::string &lens_source, const LensBuildParams &p, uint32_t *cand, std::string *err) = 0;
    // forward lenses, step 1: screen position of every plate grid point; `undecided` receives
    // the points the host has to evaluate itself
    virtual bool forward_points(const std::string &lens_source, const LensBuildParams &p, std::vector<uint32_t> *undecided, std::string *err) = 0;
    // step 2: host results patched in, quads rasterised in the reference's order (last writer
    // wins), map resolved.  messages: (order key, value) of every "%d > maxdiff" the reference prints.
    virtual bool forward_finish(const std::vector<ForwardPatch> &patches, int32_t *idx, uint8_t *tint, int display[6],
                                std::vector<std::pair<uint32_t, int>> *messages, std::string *err) = 0;
};

class LensDevice : public DeviceLensBuilder {
public:
    explicit LensDevice(int device) : device_(device) {}
    ~LensDevice() override;

    // lens_source = transpile_prelude(true) + TranspileResult::source.
    // Fills cand[width*height].  Returns false (reason in *err) when NVRTC is unavailable,
    // the source does not compile, or a CUDA call fails.
    bool build(const std::string &lens_source, const LensBuildParams &p, uint32_t *cand, std::string *err) override;
    bool forward_points(const std::string &lens_source, const LensBuildParams &p, std::vector<uint32_t> *undecided, std::string *err) override;
    bool forward_finish(const std::vector<ForwardPatch> &patches, int32_t *idx, uint8_t *tint, int display[6],
                        std::vector<std::pair<uint32_t, int>> *messages, std::string *err) override;

    // the fixed CUDA source appended to a translated lens (the per-pixel / per-grid-point tail);
    // exposed so that the CPU test-suite can run the very same text through a host shim
    static const char *kernel_tail(bool forward);

    // compile only (no GPU needed): used by the CPU test-suite and by build()
    static bool compile(const std::string &lens_source, bool forward, std::vector<char> *cubin, std::string *log);

    double last_compile_ms() const { return compile_ms_; }
    double last_kernel_ms() const { return kernel_ms_; }
    int64_t launches() const { return launches_; }

private:
    struct Module;
    struct ForwardState;
    Module *module_for(const std::string &lens_source, bool forward, std::string *err);
    void drop_forward_state();
    int device_;
    std::map<std::string, Module *> cache_;  // by flavour + source text
    ForwardState *fwd_ = nullptr;
    double compile_ms_ = 0, kernel_ms_ = 0;
    int64_t launches_ = 0;
};

}  // namespace blinky
