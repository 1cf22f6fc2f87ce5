// Device-side lensmap construction: NVRTC compile of the translated lens + launch.
// See lens_device.h.
#include "lens_device.h"
#include "forward_raster.h"

#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nvrtc.h>

#include <chrono>
#include <cstdio>
#include <cstring>
#include <mutex>

namespace blinky {

namespace {

// The per-pixel tail of the lensmap build, appended to the translated lens.  Operation
// order and types follow fisheye_host.cpp (which follows fisheye.c:2023-2066 ray_to_plate_index /
// ray_to_plate_uv, :1984-2013 set_from_ray, :1922-1960 rubix grid) line by line: after the ray is
// narrowed to float32 everything is IEEE +,-,*,/ and sqrt, compiled with --fmad=false, so it is
// bit-identical to the host.
//
// The text is kept in pieces so that a globe with a globe_plate script can replace the plate argmax
// (kernel_tail): every other globe gets exactly kKernelParams + kKernelSignature + kKernelHead + kKernelNormalize + kKernelArgmax +
// kKernelTexel + kKernelEnd.  The ray-map unit (raymap_tail) wraps the same pieces from kKernelNormalize on; the
// ray-export unit (rays_tail) puts kKernelHead, the lens half, under its own signature and end.
const char *kKernelParams = R"KRN(
struct LtParams {
    int width, height, platesize, numplates;
    double scale;
    double rubix_block, rubix_pad, rubix_unit_px;
    double uv_dist[6];
    LtPlate plates[6];
};

static __device__ __forceinline__ float lt_dot3(const float *a, const float *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
)KRN";

const char *kKernelSignature = R"KRN(
extern "C" __global__ void __launch_bounds__(128) lt_build(const __grid_constant__ LtParams P, unsigned *__restrict__ cand) {
)KRN";

// the pixel's coordinates (fisheye.c:2100-2105, integer /2) and the lens's ray, narrowed to float
const char *kKernelHead = R"KRN(    const int lx = blockIdx.x * blockDim.x + threadIdx.x, ly = blockIdx.y;
    if (lx >= P.width) return;
    const double x = (lx - P.width / 2) * P.scale;
    const double y = -(ly - P.height / 2) * P.scale;
    Ctx c;
    c.flag = 0;
    c.steps = 0;
    c.plates = P.plates;
    c.numplates = P.numplates;
    lt_init_mut(c);
    LtD r[3];
    unsigned out = 0;
    if (lt_entry(c, x, y, r)) {
        float ray[3] = {lt_f32(c, r[0]), lt_f32(c, r[1]), lt_f32(c, r[2])};
)KRN";

// normalize3 of fisheye_host.cpp (VectorNormalize)
const char *kKernelNormalize = R"KRN(        float len = ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2];
        len = (float)sqrt((double)len);
        if (len) {
            const float inv = 1 / len;
            ray[0] *= inv; ray[1] *= inv; ray[2] *= inv;
        }
)KRN";

const char *kKernelArgmax = R"KRN(        int best = 0;
        double best_dp = -2;
        for (int i = 0; i < P.numplates; ++i) {
            const double dp = (double)lt_dot3(ray, P.plates[i].forward);
            if (dp > best_dp) { best_dp = dp; best = i; }
        }
)KRN";

// ray_to_plate_index through the globe's script (fisheye.c:2027-2033) and set_from_ray's range checks:
// a plate outside 0..5 leaves the pixel unmapped; plates numplates..5 are whatever the host keeps there
const char *kKernelGlobePlateOpen = R"KRN(#ifdef LT_HAS_GLOBE_PLATE
        int best = -1;
        lt_globe_plate(c, (double)ray[0], (double)ray[1], (double)ray[2], &best);
        if (best >= 0 && best < 6) {
#else
)KRN";

const char *kKernelTexel = R"KRN(        const LtPlate &p = P.plates[best];
        const double px_ = (double)lt_dot3(p.right, ray);
        const double py_ = (double)lt_dot3(p.up, ray);
        const double pz_ = (double)lt_dot3(p.forward, ray);
        const double dist = P.uv_dist[best];
        const double u = px_ / pz_ * dist + 0.5;
        const double v = -py_ / pz_ * dist + 0.5;
        if (u >= 0 && u <= 1 && v >= 0 && v <= 1) {
            const int ps = P.platesize;
            const int px = (int)(u * ps), py = (int)(v * ps);
            if (px >= 0 && px < ps && py >= 0 && py < ps) {
                const double ux = (double)px / P.rubix_unit_px, uy = (double)py / P.rubix_unit_px;
                const bool ongrid = fmod(ux, P.rubix_block) < P.rubix_pad || fmod(uy, P.rubix_block) < P.rubix_pad;
                out = 0x80000000u | (ongrid ? 0x40000000u : 0u) | (unsigned)(best * ps * ps + px + py * ps);
            }
        }
)KRN";

const char *kKernelGlobePlateClose = R"KRN(#ifdef LT_HAS_GLOBE_PLATE
        }
#endif
)KRN";

const char *kKernelEnd = R"KRN(    }
    if (c.flag) out |= 0x20000000u;
    cand[(size_t)ly * P.width + lx] = out;
}
)KRN";

// The ray-map kernel (blinky_set_raymap_device): pixel `at` reads the caller's float32 ray instead of evaluating a lens,
// and writes its packed lensmap entry (BLINKY_LM_*) straight away: a map built in one pass gives an on-grid pixel no
// tint.  A pixel whose globe_plate decision carries a risk flag is written unmapped and listed in `flagged` for the host.
const char *kRaymapHead = R"KRN(
extern "C" __global__ void __launch_bounds__(256) lt_raymap(const __grid_constant__ LtParams P, const float *__restrict__ rays,
                                                            unsigned *__restrict__ map, unsigned *__restrict__ flagged,
                                                            unsigned *__restrict__ nflagged, unsigned flagged_cap) {
    const size_t at = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (at >= (size_t)P.width * P.height) return;
    Ctx c;
    c.flag = 0;
    c.steps = 0;
    c.plates = P.plates;
    c.numplates = P.numplates;
#ifdef LT_HAS_GLOBE_PLATE
    lt_init_mut(c);
#endif
    unsigned out = 0;
    {
        float ray[3] = {rays[3 * at], rays[3 * at + 1], rays[3 * at + 2]};
)KRN";

const char *kRaymapEnd = R"KRN(        if (out) out = (out & 0x8FFFFFFFu) | ((out & 0x40000000u) ? 7u : (unsigned)best) << 28;
    }
    if (c.flag) {
        out = 0;
        const unsigned k = atomicAdd(nflagged, 1u);
        if (k < flagged_cap) flagged[k] = (unsigned)at;
    }
    map[at] = out ? out : 0x70000000u;
}
)KRN";

// The ray-export kernel (blinky_get_raymap_device): the build's lens half (kKernelHead) for pixel (lx, ly), whose
// narrowed ray, or the zero vector for nil, goes straight into the caller's float32[height][width][3] field.  A pixel
// with a risk flag is listed in `flagged`; the host evaluates it and overwrites its ray.
const char *kRaysSignature = R"KRN(
extern "C" __global__ void __launch_bounds__(128) lt_rays(const __grid_constant__ LtParams P, float *__restrict__ rays,
                                                          unsigned *__restrict__ flagged, unsigned *__restrict__ nflagged,
                                                          unsigned flagged_cap) {
)KRN";

const char *kRaysEnd = R"KRN(        float *o = rays + 3 * ((size_t)ly * P.width + lx);
        o[0] = ray[0];
        o[1] = ray[1];
        o[2] = ray[2];
        out = 1;
    }
    const size_t at = (size_t)ly * P.width + lx;
    if (!out) rays[3 * at] = rays[3 * at + 1] = rays[3 * at + 2] = 0.0f;
    if (c.flag) {
        const unsigned k = atomicAdd(nflagged, 1u);
        if (k < flagged_cap) flagged[k] = (unsigned)at;
    }
}
)KRN";

// The math probe (blinky_probe_math, a test hook): one prelude wrapper or IEEE operation per launch, on exact
// arguments a[i] (and b[i] for the binary ones), with the prelude's value and bound.  The op numbers are
// BLINKY_PROBE_* in blinky_b200.h; modf's integral part goes to e.
const char *kProbeSource = R"KRN(
extern "C" __global__ void __launch_bounds__(256) lt_probe(int op, const double *__restrict__ a, const double *__restrict__ b,
                                                           double *__restrict__ v, double *__restrict__ e, unsigned long long n) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const LtD x(a[i]);
    LtD r(0.0);
    switch (op) {
        case 0: r = lt_sin(x); break;
        case 1: r = lt_cos(x); break;
        case 2: r = lt_tan(x); break;
        case 3: r = lt_asin(x); break;
        case 4: r = lt_acos(x); break;
        case 5: r = lt_atan(x); break;
        case 6: r = lt_atan2(x, LtD(b[i])); break;
        case 7: r = lt_exp(x); break;
        case 8: r = lt_log(x); break;
        case 9: r = lt_log10(x); break;
        case 10: r = lt_logb(x, LtD(b[i])); break;
        case 11: r = lt_sinh(x); break;
        case 12: r = lt_cosh(x); break;
        case 13: r = lt_tanh(x); break;
        case 14: r = lt_pow(x, LtD(b[i])); break;
        case 15: r = LtD(sqrt(x.v)); break;
        case 16: r = LtD(fmod(x.v, b[i])); break;
        case 17: r = LtD(floor(x.v)); break;
        case 18: r = LtD(ceil(x.v)); break;
        case 19: r = LtD(trunc(x.v)); break;
        case 20: { double ip; const double f = modf(x.v, &ip); r = LtD(f, ip); break; }
        case 21: r = LtD(x.v / b[i]); break;
        case 22: r = LtD((double)(float)x.v); break;
        case 23: r = LtD((double)(int)x.v); break;
    }
    v[i] = r.v;
    e[i] = r.e;
}
)KRN";

// Forward builder, step 1 (fisheye.c:2227-2243 uv_to_screen over the grid of fisheye.c:2151-2189):
// grid point (plate, j, i) sits at u = (i - 0.5)/ps, v = (j - 0.5)/ps.
const char *kForwardKernelSource = R"KRN(
struct LtParams {
    int width, height, platesize, numplates;
    double scale;
    double rubix_block, rubix_pad, rubix_unit_px;
    double uv_dist[6];
    LtPlate plates[6];
};

// (int) of a double with an error bound: undecided when an integer lies within the bound, or when the
// value is outside int range / NaN (x86 and CUDA convert those differently)
static __device__ __forceinline__ int lt_trunc_int(Ctx &c, LtD x) {
    if (!(fabs(x.v) < 2147483000.0)) { c.flag |= LT_RISK_NEAR; return 0; }
    if (!(x.e == 0.0)) {
        const double n = rint(x.v);
        if (!(fabs(x.v - n) > 2.0 * x.e)) c.flag |= LT_RISK_NEAR;
    }
    return (int)x.v;
}

extern "C" __global__ void __launch_bounds__(128) lt_forward_points(const __grid_constant__ LtParams P, int2 *__restrict__ grid,
                                                                    unsigned char *__restrict__ status, unsigned *__restrict__ undecided,
                                                                    unsigned *__restrict__ counters, unsigned undecided_cap) {
    const int n1 = P.platesize + 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y, plate = blockIdx.z;
    if (i >= n1) return;
    const unsigned point = ((unsigned)plate * n1 + j) * n1 + i;
    Ctx c;
    c.flag = 0;
    c.steps = 0;
    c.plates = P.plates;
    c.numplates = P.numplates;
    lt_init_mut(c);
    // plate_uv_to_ray (fisheye.c:1198-1214) for exact u, v
    double ray[3];
    lt_plate_to_ray(c, LtD((double)plate), LtD((i - 0.5) / P.platesize), LtD((j - 0.5) / P.platesize), ray);
    LtD r[2];
    int2 out = make_int2(0, 0);
    unsigned char st = 0;
    if (lt_entry(c, ray[0], ray[1], ray[2], r)) {
        st = 1;
        out.x = lt_trunc_int(c, r[0] / LtD(P.scale) + LtD((double)(P.width / 2)));
        out.y = lt_trunc_int(c, -r[1] / LtD(P.scale) + LtD((double)(P.height / 2)));
    } else {
        atomicAdd(&counters[1], 1u);   // a nil: the stale-value pass is needed
    }
    if (c.flag) {
        st = 2;
        const unsigned at = atomicAdd(&counters[0], 1u);
        if (at < undecided_cap) undecided[at] = point;
    }
    grid[point] = out;
    status[point] = st;
}
)KRN";

// Forward builder, texel owners (globes with a globe_plate script only): the texel (plate, px, py) is drawn
// only if globe_plate picks `plate` for the texel's ray (fisheye.c:2193-2199).  lt_plate_to_ray at
// u = px/ps, v = py/ps is the float arithmetic of fwd_raster_texel / plate_uv_to_ray.  One byte per texel:
// kOwnerOwned, plus kOwnerRisk (and an entry in `undecided`) where the host has to decide.
const char *kForwardOwnerKernelSource = R"KRN(
#ifdef LT_HAS_GLOBE_PLATE
extern "C" __global__ void __launch_bounds__(128) lt_forward_owner(const __grid_constant__ LtParams P, unsigned char *__restrict__ owner,
                                                                   unsigned *__restrict__ undecided, unsigned *__restrict__ counter,
                                                                   unsigned undecided_cap) {
    const int ps = P.platesize;
    const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y, plate = blockIdx.z;
    if (px >= ps) return;
    const unsigned texel = ((unsigned)plate * ps + py) * ps + px;
    Ctx c;
    c.flag = 0;
    c.steps = 0;
    c.plates = P.plates;
    c.numplates = P.numplates;
    lt_init_mut(c);
    double ray[3];
    lt_plate_to_ray(c, LtD((double)plate), LtD((double)px / ps), LtD((double)py / ps), ray);
    int sel = -1;
    lt_globe_plate(c, ray[0], ray[1], ray[2], &sel);
    unsigned char o = sel == plate ? 1 : 0;
    if (c.flag) {
        o |= 2;
        const unsigned at = atomicAdd(counter, 1u);
        if (at < undecided_cap) undecided[at] = texel;
    }
    owner[texel] = o;
}
#endif
)KRN";

struct Nvrtc {
    void *lib = nullptr;
    decltype(&nvrtcCreateProgram) CreateProgram = nullptr;
    decltype(&nvrtcCompileProgram) CompileProgram = nullptr;
    decltype(&nvrtcGetCUBINSize) GetCUBINSize = nullptr;
    decltype(&nvrtcGetCUBIN) GetCUBIN = nullptr;
    decltype(&nvrtcGetProgramLogSize) GetProgramLogSize = nullptr;
    decltype(&nvrtcGetProgramLog) GetProgramLog = nullptr;
    decltype(&nvrtcDestroyProgram) DestroyProgram = nullptr;
    decltype(&nvrtcGetErrorString) GetErrorString = nullptr;
    std::string why;
};

Nvrtc &nvrtc() {
    static Nvrtc n;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *names[] = {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12"};
        for (const char *nm : names) {
            n.lib = dlopen(nm, RTLD_NOW | RTLD_LOCAL);
            if (n.lib) break;
        }
        if (!n.lib) {
            n.why = std::string("NVRTC not found: ") + dlerror();
            return;
        }
#define LOAD(sym)                                                          \
    n.sym = reinterpret_cast<decltype(n.sym)>(dlsym(n.lib, "nvrtc" #sym)); \
    if (!n.sym) n.why = "NVRTC lacks nvrtc" #sym;
        LOAD(CreateProgram)
        LOAD(CompileProgram)
        LOAD(GetCUBINSize)
        LOAD(GetCUBIN)
        LOAD(GetProgramLogSize)
        LOAD(GetProgramLog)
        LOAD(DestroyProgram)
        LOAD(GetErrorString)
#undef LOAD
    });
    return n;
}

struct Driver {
    CUresult (*ModuleLoadData)(CUmodule *, const void *) = nullptr;
    CUresult (*ModuleGetFunction)(CUfunction *, CUmodule, const char *) = nullptr;
    CUresult (*ModuleUnload)(CUmodule) = nullptr;
    CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void **, void **) = nullptr;
    bool ok = false;
};

Driver &driver() {
    static Driver d;
    static std::once_flag once;
    std::call_once(once, [] {
        auto get = [](const char *name, void **fn) {
            cudaDriverEntryPointQueryResult q;
            return cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess && *fn;
        };
        d.ok = get("cuModuleLoadData", reinterpret_cast<void **>(&d.ModuleLoadData)) &&
               get("cuModuleGetFunction", reinterpret_cast<void **>(&d.ModuleGetFunction)) &&
               get("cuModuleUnload", reinterpret_cast<void **>(&d.ModuleUnload)) &&
               get("cuLaunchKernel", reinterpret_cast<void **>(&d.LaunchKernel));
    });
    return d;
}

}  // namespace

// one loaded unit, unloaded when its owner goes
struct LensDevice::Module {
    CUmodule mod = nullptr;
    CUfunction fn = nullptr;
    CUfunction owner_fn = nullptr;  // forward modules of globes with a globe_plate script
    Module() = default;
    Module(const Module &) = delete;
    Module &operator=(const Module &) = delete;
    ~Module() {
        if (mod) driver().ModuleUnload(mod);
    }
};

// device buffers that live between forward_points() and forward_finish()
struct LensDevice::ForwardState {
    LensBuildParams p;
    DeviceBuffer grid;       // FwdPoint[npoints]
    DeviceBuffer status;     // unsigned char[npoints]
    DeviceBuffer undecided;  // unsigned[kUndecidedCap]
    DeviceBuffer counters;   // unsigned[16]: [0] undecided points, [1] nil results, [2] messages, [3..8] display flags, [9] undecided owners
    unsigned nil_count = 0;
    DeviceBuffer owner;            // [numplates * ps * ps] texel owners; empty: the plate argmax decides
    DeviceBuffer owner_undecided;  // unsigned[kUndecidedCap]
    // from patch_forward on
    DeviceBuffer keys;             // idxkey[npix] then tintkey[npix]
    DeviceBuffer messages;         // FwdMessage[kFwdMessageCap]
    DeviceBuffer patches, owner_patches;  // the host's grid points and texel owners
    bool any_nil = false;          // a grid point is nil: the stale slots need replaying
};

namespace {

constexpr unsigned kUndecidedCap = 1u << 20;
constexpr unsigned kMessageCap = kFwdMessageCap;

// ---- forward builder, steps 2-4 (this file is compiled with --fmad=false) ---------------------------
// The per-thread bodies live in forward_raster.h (host/device) so that the CPU suite can run them
// — in arbitrary thread orders — against the reference-equivalent serial builder.

__global__ void fwd_patch_kernel(FwdPoint *grid, unsigned char *status, const ForwardPatch *patches, unsigned n) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) fwd_apply_patch(grid, status, patches[k]);
}

__global__ void fwd_stale_kernel(FwdPoint *grid, const unsigned char *status, int ps, int numplates) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < 2 * (ps + 1)) fwd_stale_chain(grid, status, ps, numplates, t);
}

__global__ void fwd_owner_patch_kernel(unsigned char *owner, const uint32_t *patches, unsigned n) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) fwd_apply_owner_patch(owner, patches[k]);
}

// the rays of the listed pixels, for the host to settle (ray maps)
__global__ void gather_rays_kernel(const float *__restrict__ rays, const unsigned *__restrict__ pixels, unsigned n, float *__restrict__ out) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const size_t at = pixels[k];
    for (int i = 0; i < 3; ++i) out[3 * k + i] = rays[3 * at + i];
}

__global__ void scatter_entries_kernel(uint32_t *__restrict__ map, const RayPatch *__restrict__ patches, unsigned n) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) map[patches[k].pixel] = patches[k].entry;
}

// the rays the host evaluated, into the exported field (ray export)
__global__ void scatter_rays_kernel(float *__restrict__ rays, const RaySample *__restrict__ samples, unsigned n) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const size_t at = samples[k].pixel;
    for (int i = 0; i < 3; ++i) rays[3 * at + i] = samples[k].ray[i];
}

__global__ void __launch_bounds__(128) fwd_raster_kernel(const __grid_constant__ FwdGeom g, const FwdPoint *__restrict__ grid, FwdOut o,
                                                         const unsigned char *__restrict__ owner) {
    const int px = blockIdx.x * blockDim.x + threadIdx.x;
    if (px < g.ps) fwd_raster_texel(g, grid, o, static_cast<int>(blockIdx.z), static_cast<int>(blockIdx.y), px, owner);
}

__global__ void fwd_resolve_kernel(const unsigned *__restrict__ idxkey, const unsigned *__restrict__ tintkey, int32_t *__restrict__ idx,
                                   uint8_t *__restrict__ tint, size_t npix, int ps) {
    const size_t at = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (at < npix) fwd_resolve_pixel(idxkey, tintkey, idx, tint, at, ps);
}

// the exported ray of each pixel from the forward build's winning texel (ray export of a forward lens, DESIGN §3h)
__global__ void __launch_bounds__(256) fwd_ray_kernel(const __grid_constant__ FwdGeom g, const FwdPoint *__restrict__ grid,
                                                      const unsigned *__restrict__ idxkey, float *__restrict__ rays, size_t npix) {
    const size_t at = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (at >= npix) return;
    const int y = static_cast<int>(at / static_cast<unsigned>(g.width)), x = static_cast<int>(at - static_cast<size_t>(y) * g.width);
    float r[3];
    fwd_ray_pixel(g, grid, idxkey[at], x, y, r);
    rays[3 * at] = r[0];
    rays[3 * at + 1] = r[1];
    rays[3 * at + 2] = r[2];
}

// true when ce is cudaSuccess; otherwise false with "what: <CUDA error>" in *err
bool checked(cudaError_t ce, const char *what, std::string *err) {
    if (ce != cudaSuccess) *err = std::string(what) + ": " + cudaGetErrorString(ce);
    return ce == cudaSuccess;
}

cudaError_t allocate(DeviceBuffer *b, size_t bytes) { return static_cast<cudaError_t>(b->alloc(bytes)); }

// a device copy of v, copied on `s`: the caller synchronises `s` before v may change or go
template <typename T>
DeviceBuffer upload(const std::vector<T> &v, cudaStream_t s, cudaError_t *ce) {
    DeviceBuffer d;
    *ce = allocate(&d, v.size() * sizeof(T));
    if (*ce == cudaSuccess) *ce = cudaMemcpyAsync(d.get(), v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s);
    return d;
}

// launches a kernel of a compiled unit, `block` threads per block, on `s`
bool launch(CUfunction fn, dim3 grid, unsigned block, cudaStream_t s, void **args, std::string *err) {
    const CUresult cr = driver().LaunchKernel(fn, grid.x, grid.y, grid.z, block, 1, 1, 0, s, args, nullptr);
    if (cr != CUDA_SUCCESS) *err = "cuLaunchKernel failed (CUresult " + std::to_string(static_cast<int>(cr)) + ")";
    return cr == CUDA_SUCCESS;
}

// A list a kernel filled for the host, read back on `s`: the count at d_count, then that many entries of d_list, into
// *out.  False with the reason in *err on a CUDA error (what: the kernel, for the message) or when more than
// kUndecidedCap items (a plural noun) need the interpreter.
bool read_list(const unsigned *d_count, const unsigned *d_list, cudaStream_t s, const char *what, const char *items,
               std::vector<uint32_t> *out, std::string *err) {
    unsigned n = 0;
    cudaError_t ce = cudaMemcpyAsync(&n, d_count, sizeof n, cudaMemcpyDeviceToHost, s);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
    if (!checked(ce, what, err)) return false;
    if (n > kUndecidedCap) {
        *err = std::string("too many ") + items + " need the interpreter (" + std::to_string(n) + ")";
        return false;
    }
    out->resize(n);
    if (n == 0) return true;
    ce = cudaMemcpyAsync(out->data(), d_list, n * sizeof(unsigned), cudaMemcpyDeviceToHost, s);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
    return checked(ce, what, err);
}

// two events around a window of work on one stream
class EventTimer {
public:
    EventTimer() {
        created_ = cudaEventCreate(&begin_);
        if (created_ == cudaSuccess) created_ = cudaEventCreate(&end_);
    }
    EventTimer(const EventTimer &) = delete;
    EventTimer &operator=(const EventTimer &) = delete;
    ~EventTimer() {
        if (begin_) cudaEventDestroy(begin_);
        if (end_) cudaEventDestroy(end_);
    }
    // opens the window: the error of creating the events or of recording the first
    cudaError_t start(cudaStream_t s) { return created_ == cudaSuccess ? cudaEventRecord(begin_, s) : created_; }
    void stop(cudaStream_t s) { cudaEventRecord(end_, s); }
    // the window's milliseconds, once the stream is past stop()
    float ms() const {
        float ms = 0;
        cudaEventElapsedTime(&ms, begin_, end_);
        return ms;
    }

private:
    cudaEvent_t begin_ = nullptr, end_ = nullptr;
    cudaError_t created_;
};

}  // namespace

LensDevice::LensDevice(int device) : device_(device) {}

LensDevice::~LensDevice() = default;

std::string LensDevice::kernel_tail(bool forward, bool globe_plate) {
    if (forward) return globe_plate ? std::string(kForwardKernelSource) + kForwardOwnerKernelSource : std::string(kForwardKernelSource);
    const std::string head = std::string(kKernelParams) + kKernelSignature + kKernelHead + kKernelNormalize;
    if (!globe_plate) return head + kKernelArgmax + kKernelTexel + kKernelEnd;
    return head + kKernelGlobePlateOpen + kKernelArgmax + "#endif\n" + kKernelTexel + kKernelGlobePlateClose + kKernelEnd;
}

std::string LensDevice::rays_tail() { return std::string(kKernelParams) + kRaysSignature + kKernelHead + kRaysEnd; }

std::string LensDevice::probe_tail() { return kProbeSource; }

std::string LensDevice::raymap_tail(bool globe_plate) {
    const std::string head = std::string(kKernelParams) + kRaymapHead + kKernelNormalize;
    if (!globe_plate) return head + kKernelArgmax + kKernelTexel + kRaymapEnd;
    return head + kKernelGlobePlateOpen + kKernelArgmax + "#endif\n" + kKernelTexel + kKernelGlobePlateClose + kRaymapEnd;
}

bool LensDevice::compile(const std::string &lens_source, bool forward, std::vector<char> *cubin, std::string *log) {
    return compile_unit(lens_source + kernel_tail(forward, source_has_globe_plate(lens_source)), cubin, log);
}

bool LensDevice::compile_unit(const std::string &src, std::vector<char> *cubin, std::string *log) {
    Nvrtc &n = nvrtc();
    if (!n.why.empty()) {
        *log = n.why;
        return false;
    }
    nvrtcProgram prog;
    nvrtcResult rc = n.CreateProgram(&prog, src.c_str(), "lens.cu", 0, nullptr, nullptr);
    if (rc != NVRTC_SUCCESS) {
        *log = std::string("nvrtcCreateProgram: ") + n.GetErrorString(rc);
        return false;
    }
    // --fmad=false: the host computes with -ffp-contract=off; parity needs unfused arithmetic
    const char *opts[] = {"--gpu-architecture=sm_90a", "--fmad=false", "--std=c++17", "--prec-div=true", "--prec-sqrt=true", "--ftz=false", "--disable-warnings"};
    rc = n.CompileProgram(prog, static_cast<int>(sizeof(opts) / sizeof(opts[0])), opts);
    size_t logsz = 0;
    n.GetProgramLogSize(prog, &logsz);
    if (logsz > 1) {
        log->resize(logsz);
        n.GetProgramLog(prog, &(*log)[0]);
    }
    if (rc != NVRTC_SUCCESS) {
        *log = std::string("NVRTC: ") + n.GetErrorString(rc) + "\n" + *log;
        n.DestroyProgram(&prog);
        return false;
    }
    size_t sz = 0;
    n.GetCUBINSize(prog, &sz);
    cubin->resize(sz);
    n.GetCUBIN(prog, cubin->data());
    n.DestroyProgram(&prog);
    return sz > 0;
}

LensDevice::Module *LensDevice::module_for(const std::string &source, Unit unit, std::string *err) {
    // per unit (in Unit's order): the letter of its cache keys, the kernel it launches and the tail appended to source
    static const struct {
        char key;
        const char *entry;
        std::string (*tail)(const std::string &source);
    } kUnits[] = {
        {'I', "lt_build", [](const std::string &s) { return kernel_tail(false, source_has_globe_plate(s)); }},
        {'F', "lt_forward_points", [](const std::string &s) { return kernel_tail(true, source_has_globe_plate(s)); }},
        {'R', "lt_raymap", [](const std::string &s) { return raymap_tail(source_has_globe_plate(s)); }},
        {'E', "lt_rays", [](const std::string &) { return rays_tail(); }},
        {'P', "lt_probe", [](const std::string &) { return probe_tail(); }},
    };
    const auto &u = kUnits[unit];
    compile_ms_ = 0;
    // (since CUDA 12 this also makes the device's primary context current, which cuModuleLoadData needs)
    if (cudaSetDevice(device_) != cudaSuccess) {
        *err = "cudaSetDevice failed";
        return nullptr;
    }
    Driver &d = driver();
    if (!d.ok) {
        *err = "CUDA driver entry points unavailable";
        return nullptr;
    }
    const std::string cache_key = u.key + source;
    auto it = cache_.find(cache_key);
    if (it != cache_.end()) return it->second.get();
    auto t0 = std::chrono::steady_clock::now();
    std::vector<char> cubin;
    std::string log;
    if (!compile_unit(source + u.tail(source), &cubin, &log)) {
        *err = log;
        return nullptr;
    }
    auto m = std::make_unique<Module>();
    CUresult cr = d.ModuleLoadData(&m->mod, cubin.data());
    if (cr == CUDA_SUCCESS) cr = d.ModuleGetFunction(&m->fn, m->mod, u.entry);
    if (cr == CUDA_SUCCESS && unit == kForwardUnit && source_has_globe_plate(source)) cr = d.ModuleGetFunction(&m->owner_fn, m->mod, "lt_forward_owner");
    if (cr != CUDA_SUCCESS) {
        *err = "loading the compiled lens failed (CUresult " + std::to_string(static_cast<int>(cr)) + ")";
        return nullptr;
    }
    if (cache_.size() >= 16) cache_.clear();  // lenses are few; keep the cache from growing without bound
    Module *loaded = m.get();
    cache_[cache_key] = std::move(m);
    compile_ms_ = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return loaded;
}

bool LensDevice::build(const std::string &lens_source, const LensBuildParams &p, uint32_t *cand, std::string *err) {
    kernel_ms_ = 0;
    if (p.height > 65535) {   // one row of blocks per screen row, and gridDim.y is at most 65535
        *err = "screen taller than 65535 rows, the device lens kernel's grid limit";
        return false;
    }
    Module *m = module_for(lens_source, kInverseUnit, err);
    if (!m) return false;
    const size_t npix = static_cast<size_t>(p.width) * p.height;
    DeviceBuffer d_cand;
    if (!checked(allocate(&d_cand, npix * sizeof(uint32_t)), "cudaMalloc", err)) return false;
    EventTimer timer;
    if (!checked(timer.start(nullptr), "lens kernel", err)) return false;
    LensBuildParams params = p;
    uint32_t *out = d_cand.as<uint32_t>();
    void *args[] = {&params, &out};
    const unsigned block = 128;
    if (!launch(m->fn, dim3((p.width + block - 1) / block, p.height), block, nullptr, args, err)) return false;
    timer.stop(nullptr);
    if (!checked(cudaMemcpy(cand, out, npix * sizeof(uint32_t), cudaMemcpyDeviceToHost), "lens kernel", err)) return false;  // synchronises
    kernel_ms_ = timer.ms();
    return true;
}

bool LensDevice::raymap(const std::string &globe_source, const LensBuildParams &p, const float *d_rays, void *stream, uint32_t **d_map,
                        std::vector<uint32_t> *flagged, std::vector<float> *flagged_rays, std::string *err) {
    kernel_ms_ = 0;
    const size_t npix = static_cast<size_t>(p.width) * p.height;
    if (npix >= 0xFFFFFFFFull) {   // the flagged list holds 32-bit pixel numbers
        *err = "screen of 2^32 pixels or more";
        return false;
    }
    Module *m = module_for(globe_source, kRaymapUnit, err);
    if (!m) return false;
    // kept for the context's later ray maps: the look-around loop makes one per frame
    cudaError_t ce = cudaSuccess;
    if (!ray_flagged_.get()) ce = allocate(&ray_flagged_, (1 + static_cast<size_t>(kUndecidedCap)) * sizeof(unsigned));
    if (ce == cudaSuccess && ray_map_pixels_ < npix) {
        ray_map_pixels_ = 0;
        ce = allocate(&ray_map_, npix * sizeof(uint32_t));
        if (ce == cudaSuccess) ray_map_pixels_ = npix;
    }
    if (!checked(ce, "cudaMalloc", err)) return false;
    uint32_t *map = ray_map_.as<uint32_t>();
    *d_map = map;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    EventTimer timer;
    LensBuildParams params = p;
    unsigned *count = ray_flagged_.as<unsigned>(), *list = count + 1;
    unsigned cap = kUndecidedCap;
    void *args[] = {&params, &d_rays, &map, &list, &count, &cap};
    const unsigned block = 256;
    ce = cudaMemsetAsync(count, 0, sizeof(unsigned), s);
    if (ce == cudaSuccess) ce = timer.start(s);
    if (!checked(ce, "ray map kernel", err)) return false;
    if (!launch(m->fn, dim3(static_cast<unsigned>((npix + block - 1) / block)), block, s, args, err)) return false;
    timer.stop(s);
    if (!read_list(count, list, s, "ray map kernel", "pixels", flagged, err)) return false;
    kernel_ms_ = timer.ms();
    const unsigned n = static_cast<unsigned>(flagged->size());
    flagged_rays->resize(3 * static_cast<size_t>(n));
    if (n == 0) return true;
    // only the flagged pixels' rays come back
    DeviceBuffer d_gathered;
    ce = allocate(&d_gathered, flagged_rays->size() * sizeof(float));
    if (ce == cudaSuccess) {
        gather_rays_kernel<<<(n + 255) / 256, 256, 0, s>>>(d_rays, list, n, d_gathered.as<float>());
        ce = cudaMemcpyAsync(flagged_rays->data(), d_gathered.get(), flagged_rays->size() * sizeof(float), cudaMemcpyDeviceToHost, s);
    }
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
    return checked(ce, "ray map gather", err);
}

bool LensDevice::patch_entries(const std::vector<RayPatch> &patches, void *stream, std::string *err) {
    if (patches.empty()) return true;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    cudaError_t ce;
    const DeviceBuffer d_patches = upload(patches, s, &ce);
    if (ce == cudaSuccess) {
        const unsigned n = static_cast<unsigned>(patches.size());
        scatter_entries_kernel<<<(n + 255) / 256, 256, 0, s>>>(ray_map_.as<uint32_t>(), d_patches.as<RayPatch>(), n);
        ce = cudaStreamSynchronize(s);  // (patches is pageable host memory the copy may still read)
    }
    return checked(ce, "ray map patch", err);
}

bool LensDevice::copy_to_host(void *dst, const void *d_src, size_t bytes, void *stream, std::string *err) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    cudaError_t ce = cudaSetDevice(device_);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, s);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
    return checked(ce, "copying the rays to the host", err);
}

bool LensDevice::copy_to_device(void *d_dst, const void *src, size_t bytes, void *stream, std::string *err) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    cudaError_t ce = cudaSetDevice(device_);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyHostToDevice, s);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);  // (src is pageable host memory the copy may still read)
    return checked(ce, "copying the rays to the device", err);
}

bool LensDevice::capturing(void *stream) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    // an error (the legacy stream while another stream captures) counts as capturing: the call could not synchronise
    return cudaStreamIsCapturing(static_cast<cudaStream_t>(stream), &st) != cudaSuccess || st != cudaStreamCaptureStatusNone;
}

bool LensDevice::probe_math(const std::string &prelude, int op, const double *d_a, const double *d_b, double *d_v, double *d_e, size_t n,
                            void *stream, std::string *err) {
    Module *m = module_for(prelude, kProbeUnit, err);
    if (!m) return false;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    unsigned long long count = n;
    void *args[] = {&op, &d_a, &d_b, &d_v, &d_e, &count};
    const unsigned block = 256;
    if (!launch(m->fn, dim3(static_cast<unsigned>((n + block - 1) / block)), block, s, args, err)) return false;
    return checked(cudaStreamSynchronize(s), "math probe", err);
}

bool LensDevice::rays(const std::string &lens_source, const LensBuildParams &p, float *d_rays, void *stream, std::vector<uint32_t> *flagged,
                      std::string *err) {
    kernel_ms_ = 0;
    if (p.height > 65535) {   // one row of blocks per screen row, as lt_build
        *err = "screen taller than 65535 rows, the device lens kernel's grid limit";
        return false;
    }
    if (static_cast<size_t>(p.width) * p.height >= 0xFFFFFFFFull) {   // the flagged list holds 32-bit pixel numbers
        *err = "screen of 2^32 pixels or more";
        return false;
    }
    Module *m = module_for(lens_source, kRaysUnit, err);
    if (!m) return false;
    if (!ray_flagged_.get() && !checked(allocate(&ray_flagged_, (1 + static_cast<size_t>(kUndecidedCap)) * sizeof(unsigned)), "cudaMalloc", err))
        return false;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    EventTimer timer;
    LensBuildParams params = p;
    unsigned *count = ray_flagged_.as<unsigned>(), *list = count + 1;
    unsigned cap = kUndecidedCap;
    void *args[] = {&params, &d_rays, &list, &count, &cap};
    const unsigned block = 128;
    cudaError_t ce = cudaMemsetAsync(count, 0, sizeof(unsigned), s);
    if (ce == cudaSuccess) ce = timer.start(s);
    if (!checked(ce, "ray export kernel", err)) return false;
    if (!launch(m->fn, dim3((p.width + block - 1) / block, p.height), block, s, args, err)) return false;
    timer.stop(s);
    if (!read_list(count, list, s, "ray export kernel", "pixels", flagged, err)) return false;
    kernel_ms_ = timer.ms();
    return true;
}

bool LensDevice::patch_rays(const std::vector<RaySample> &samples, float *d_rays, void *stream, std::string *err) {
    if (samples.empty()) return true;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    cudaError_t ce;
    const DeviceBuffer d_samples = upload(samples, s, &ce);
    if (ce == cudaSuccess) {
        const unsigned n = static_cast<unsigned>(samples.size());
        scatter_rays_kernel<<<(n + 255) / 256, 256, 0, s>>>(d_rays, d_samples.as<RaySample>(), n);
        ce = cudaStreamSynchronize(s);  // (samples is pageable host memory the copy may still read)
    }
    return checked(ce, "ray export patch", err);
}

bool LensDevice::forward_points(const std::string &lens_source, const LensBuildParams &p, std::vector<uint32_t> *undecided,
                                std::vector<uint32_t> *undecided_texels, std::string *err) {
    undecided_texels->clear();
    kernel_ms_ = 0;
    fwd_.reset();
    Module *m = module_for(lens_source, kForwardUnit, err);
    if (!m) return false;
    const size_t n1 = static_cast<size_t>(p.platesize) + 1;
    const size_t npoints = static_cast<size_t>(p.numplates) * n1 * n1;
    if (npoints >= 0xFFFFFFFFull) {
        *err = "too many grid points";
        return false;
    }
    auto f = std::make_unique<ForwardState>();
    f->p = p;
    cudaError_t ce = allocate(&f->grid, npoints * sizeof(FwdPoint));
    if (ce == cudaSuccess) ce = allocate(&f->status, npoints);
    if (ce == cudaSuccess) ce = allocate(&f->undecided, kUndecidedCap * sizeof(unsigned));
    if (ce == cudaSuccess) ce = allocate(&f->counters, 16 * sizeof(unsigned));
    if (ce == cudaSuccess) ce = cudaMemset(f->counters.get(), 0, 16 * sizeof(unsigned));
    const size_t ntexels = static_cast<size_t>(p.numplates) * p.platesize * p.platesize;
    if (m->owner_fn) {
        if (ce == cudaSuccess) ce = allocate(&f->owner, ntexels);
        if (ce == cudaSuccess) ce = allocate(&f->owner_undecided, kUndecidedCap * sizeof(unsigned));
    }
    if (!checked(ce, "cudaMalloc", err)) return false;
    EventTimer timer;
    if (!checked(timer.start(nullptr), "lens kernel", err)) return false;
    LensBuildParams params = p;
    unsigned cap = kUndecidedCap;
    FwdPoint *grid = f->grid.as<FwdPoint>();
    unsigned char *status = f->status.as<unsigned char>(), *owner = f->owner.as<unsigned char>();
    unsigned *counters = f->counters.as<unsigned>(), *points = f->undecided.as<unsigned>(), *texels = f->owner_undecided.as<unsigned>();
    void *args[] = {&params, &grid, &status, &points, &counters, &cap};
    const unsigned block = 128;
    if (!launch(m->fn, dim3(static_cast<unsigned>((n1 + block - 1) / block), static_cast<unsigned>(n1), static_cast<unsigned>(p.numplates)), block,
                nullptr, args, err))
        return false;
    if (m->owner_fn) {
        unsigned *owner_counter = counters + 9;
        void *oargs[] = {&params, &owner, &texels, &owner_counter, &cap};
        const unsigned ps = static_cast<unsigned>(p.platesize);
        if (!launch(m->owner_fn, dim3((ps + block - 1) / block, ps, static_cast<unsigned>(p.numplates)), block, nullptr, oargs, err)) return false;
    }
    timer.stop(nullptr);
    if (!read_list(counters, points, nullptr, "lens kernel", "grid points", undecided, err)) return false;
    if (m->owner_fn && !read_list(counters + 9, texels, nullptr, "lens kernel", "texel owners", undecided_texels, err)) return false;
    if (!checked(cudaMemcpy(&f->nil_count, counters + 1, sizeof(unsigned), cudaMemcpyDeviceToHost), "lens kernel", err)) return false;
    kernel_ms_ = timer.ms();
    fwd_ = std::move(f);
    return true;
}

bool LensDevice::patch_forward(ForwardState &f, const std::vector<ForwardPatch> &patches, const std::vector<uint32_t> &owner_patches,
                               void *stream, std::string *err) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t npix = static_cast<size_t>(f.p.width) * f.p.height;
    cudaError_t ce = allocate(&f.keys, 2 * npix * sizeof(unsigned));
    if (ce == cudaSuccess) ce = cudaMemsetAsync(f.keys.get(), 0, 2 * npix * sizeof(unsigned), s);
    if (ce == cudaSuccess) ce = allocate(&f.messages, kMessageCap * sizeof(FwdMessage));
    FwdPoint *grid = f.grid.as<FwdPoint>();
    unsigned char *status = f.status.as<unsigned char>(), *owner = f.owner.as<unsigned char>();
    f.any_nil = f.nil_count > 0;
    if (ce == cudaSuccess && !patches.empty()) {
        f.patches = upload(patches, s, &ce);
        if (ce == cudaSuccess) {
            const unsigned n = static_cast<unsigned>(patches.size());
            fwd_patch_kernel<<<(n + 255) / 256, 256, 0, s>>>(grid, status, f.patches.as<ForwardPatch>(), n);
        }
        for (const ForwardPatch &pt : patches) f.any_nil = f.any_nil || pt.status != 1;
    }
    if (ce == cudaSuccess && !owner_patches.empty() && owner) {
        f.owner_patches = upload(owner_patches, s, &ce);
        if (ce == cudaSuccess) {
            const unsigned n = static_cast<unsigned>(owner_patches.size());
            fwd_owner_patch_kernel<<<(n + 255) / 256, 256, 0, s>>>(owner, f.owner_patches.as<uint32_t>(), n);
        }
    }
    return checked(ce, "forward lensmap kernels", err);
}

namespace {

FwdGeom forward_geom(const LensBuildParams &p) {
    FwdGeom g;
    g.width = p.width;
    g.height = p.height;
    g.ps = p.platesize;
    g.numplates = p.numplates;
    g.rubix_block = p.rubix_block;
    g.rubix_pad = p.rubix_pad;
    g.rubix_unit_px = p.rubix_unit_px;
    memcpy(g.plates, p.plates, sizeof g.plates);
    return g;
}

}  // namespace

void LensDevice::raster_forward(ForwardState &f, void *stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const LensBuildParams &p = f.p;
    const size_t npix = static_cast<size_t>(p.width) * p.height;
    FwdPoint *grid = f.grid.as<FwdPoint>();
    unsigned char *status = f.status.as<unsigned char>(), *owner = f.owner.as<unsigned char>();
    if (f.any_nil) {
        const int threads = 2 * (p.platesize + 1);
        fwd_stale_kernel<<<(threads + 63) / 64, 64, 0, s>>>(grid, status, p.platesize, p.numplates);
    }
    unsigned *keys = f.keys.as<unsigned>();
    FwdOut o{keys, keys + npix, f.counters.as<unsigned>(), f.messages.as<FwdMessage>()};
    dim3 blocks((p.platesize + 127) / 128, p.platesize, p.numplates);
    fwd_raster_kernel<<<blocks, 128, 0, s>>>(forward_geom(p), grid, o, owner);
}

bool LensDevice::forward_finish(const std::vector<ForwardPatch> &patches, const std::vector<uint32_t> &owner_patches, int32_t *idx,
                                uint8_t *tint, int display[6], std::vector<std::pair<uint32_t, int>> *messages, std::string *err) {
    const std::unique_ptr<ForwardState> f = std::move(fwd_);  // consumed whatever the outcome
    if (!f) {
        *err = "forward_finish without forward_points";
        return false;
    }
    const LensBuildParams &p = f->p;
    const size_t npix = static_cast<size_t>(p.width) * p.height;
    DeviceBuffer d_idx, d_tint;
    if (!patch_forward(*f, patches, owner_patches, nullptr, err)) return false;
    cudaError_t ce = allocate(&d_idx, npix * sizeof(int32_t));
    if (ce == cudaSuccess) ce = allocate(&d_tint, npix);
    EventTimer timer;
    if (ce == cudaSuccess) ce = timer.start(nullptr);
    if (ce == cudaSuccess) {
        raster_forward(*f, nullptr);
        unsigned *keys = f->keys.as<unsigned>();
        fwd_resolve_kernel<<<static_cast<unsigned>((npix + 255) / 256), 256>>>(keys, keys + npix, d_idx.as<int32_t>(), d_tint.as<uint8_t>(), npix, p.platesize);
        timer.stop(nullptr);
        ce = cudaMemcpy(idx, d_idx.get(), npix * sizeof(int32_t), cudaMemcpyDeviceToHost);
        if (ce == cudaSuccess) ce = cudaMemcpy(tint, d_tint.get(), npix, cudaMemcpyDeviceToHost);
    }
    unsigned counters[16] = {};
    if (ce == cudaSuccess) ce = cudaMemcpy(counters, f->counters.get(), sizeof counters, cudaMemcpyDeviceToHost);
    if (!checked(ce, "forward lensmap kernels", err)) return false;
    if (counters[2] > kMessageCap) {
        *err = "too many 'maxdiff' messages to replay (" + std::to_string(counters[2]) + ")";
        return false;
    }
    kernel_ms_ += timer.ms();
    for (int i = 0; i < 6; ++i) display[i] = counters[3 + i] ? 1 : 0;
    std::vector<FwdMessage> msg(counters[2]);
    if (counters[2] && !checked(cudaMemcpy(msg.data(), f->messages.get(), counters[2] * sizeof(FwdMessage), cudaMemcpyDeviceToHost),
                                "forward lensmap kernels", err))
        return false;
    messages->clear();
    for (const FwdMessage &m : msg) messages->emplace_back(m.key, static_cast<int>(m.value));
    return true;
}

bool LensDevice::forward_rays(const std::vector<ForwardPatch> &patches, const std::vector<uint32_t> &owner_patches, float *d_rays, void *stream,
                              std::string *err) {
    const std::unique_ptr<ForwardState> f = std::move(fwd_);  // consumed whatever the outcome
    ray_kernel_ms_ = 0;
    if (!f) {
        *err = "forward_rays without forward_points";
        return false;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const LensBuildParams &p = f->p;
    const size_t npix = static_cast<size_t>(p.width) * p.height;
    if (!patch_forward(*f, patches, owner_patches, stream, err)) return false;
    EventTimer timer, ray_timer;
    cudaError_t ce = timer.start(s);
    if (ce == cudaSuccess) {
        raster_forward(*f, stream);
        ce = ray_timer.start(s);
    }
    if (ce == cudaSuccess) {
        const unsigned block = 256;
        fwd_ray_kernel<<<static_cast<unsigned>((npix + block - 1) / block), block, 0, s>>>(forward_geom(p), f->grid.as<FwdPoint>(), f->keys.as<unsigned>(),
                                                                                          d_rays, npix);
        ce = cudaGetLastError();
        ray_timer.stop(s);
        timer.stop(s);
    }
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);  // (the patches are pageable host memory the copies may still read)
    if (!checked(ce, "forward ray export kernels", err)) return false;
    kernel_ms_ += timer.ms();
    ray_kernel_ms_ = ray_timer.ms();
    return true;
}

}  // namespace blinky
