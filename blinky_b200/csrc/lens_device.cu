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
const char *kKernelSource = R"KRN(
struct LtParams {
    int width, height, platesize, numplates;
    double scale;
    double rubix_block, rubix_pad, rubix_unit_px;
    double uv_dist[6];
    LtPlate plates[6];
};

static __device__ __forceinline__ float lt_dot3(const float *a, const float *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

extern "C" __global__ void __launch_bounds__(128) lt_build(const __grid_constant__ LtParams P, unsigned *__restrict__ cand) {
    const int lx = blockIdx.x * blockDim.x + threadIdx.x, ly = blockIdx.y;
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
        float len = ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2];
        len = (float)sqrt((double)len);
        if (len) {
            const float inv = 1 / len;
            ray[0] *= inv; ray[1] *= inv; ray[2] *= inv;
        }
        int best = 0;
        double best_dp = -2;
        for (int i = 0; i < P.numplates; ++i) {
            const double dp = (double)lt_dot3(ray, P.plates[i].forward);
            if (dp > best_dp) { best_dp = dp; best = i; }
        }
        const LtPlate &p = P.plates[best];
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
    }
    if (c.flag) out |= 0x20000000u;
    cand[(size_t)ly * P.width + lx] = out;
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

struct LensDevice::Module {
    CUmodule mod = nullptr;
    CUfunction fn = nullptr;
};

// device buffers that live between forward_points() and forward_finish()
struct LensDevice::ForwardState {
    LensBuildParams p;
    size_t npoints = 0;
    FwdPoint *grid = nullptr;
    unsigned char *status = nullptr;
    unsigned *undecided = nullptr;
    unsigned *counters = nullptr;  // [0] undecided points, [1] nil results, [2] messages, [3..8] display flags
    unsigned nil_count = 0;
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

__global__ void __launch_bounds__(128) fwd_raster_kernel(const __grid_constant__ FwdGeom g, const FwdPoint *__restrict__ grid, FwdOut o) {
    const int px = blockIdx.x * blockDim.x + threadIdx.x;
    if (px < g.ps) fwd_raster_texel(g, grid, o, static_cast<int>(blockIdx.z), static_cast<int>(blockIdx.y), px);
}

__global__ void fwd_resolve_kernel(const unsigned *__restrict__ idxkey, const unsigned *__restrict__ tintkey, int32_t *__restrict__ idx,
                                   uint8_t *__restrict__ tint, size_t npix, int ps) {
    const size_t at = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (at < npix) fwd_resolve_pixel(idxkey, tintkey, idx, tint, at, ps);
}

}  // namespace

LensDevice::~LensDevice() {
    drop_forward_state();
    for (auto &kv : cache_) {
        if (kv.second->mod && driver().ok) driver().ModuleUnload(kv.second->mod);
        delete kv.second;
    }
}

void LensDevice::drop_forward_state() {
    if (!fwd_) return;
    cudaFree(fwd_->grid);
    cudaFree(fwd_->status);
    cudaFree(fwd_->undecided);
    cudaFree(fwd_->counters);
    delete fwd_;
    fwd_ = nullptr;
}

const char *LensDevice::kernel_tail(bool forward) { return forward ? kForwardKernelSource : kKernelSource; }

bool LensDevice::compile(const std::string &lens_source, bool forward, std::vector<char> *cubin, std::string *log) {
    Nvrtc &n = nvrtc();
    if (!n.why.empty()) {
        *log = n.why;
        return false;
    }
    const std::string src = lens_source + (forward ? kForwardKernelSource : kKernelSource);
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

LensDevice::Module *LensDevice::module_for(const std::string &lens_source, bool forward, std::string *err) {
    compile_ms_ = 0;
    if (cudaSetDevice(device_) != cudaSuccess) {
        *err = "cudaSetDevice failed";
        return nullptr;
    }
    Driver &d = driver();
    if (!d.ok) {
        *err = "CUDA driver entry points unavailable";
        return nullptr;
    }
    const std::string cache_key = (forward ? "F" : "I") + lens_source;
    auto it = cache_.find(cache_key);
    if (it != cache_.end()) return it->second;
    auto t0 = std::chrono::steady_clock::now();
    std::vector<char> cubin;
    std::string log;
    if (!compile(lens_source, forward, &cubin, &log)) {
        *err = log;
        return nullptr;
    }
    cudaFree(nullptr);  // make sure the primary context is current
    Module *m = new Module;
    CUresult cr = d.ModuleLoadData(&m->mod, cubin.data());
    if (cr == CUDA_SUCCESS) cr = d.ModuleGetFunction(&m->fn, m->mod, forward ? "lt_forward_points" : "lt_build");
    if (cr != CUDA_SUCCESS) {
        if (m->mod) d.ModuleUnload(m->mod);
        delete m;
        *err = "loading the compiled lens failed (CUresult " + std::to_string(static_cast<int>(cr)) + ")";
        return nullptr;
    }
    if (cache_.size() >= 16) {  // lenses are few; keep the cache from growing without bound
        for (auto &kv : cache_) {
            d.ModuleUnload(kv.second->mod);
            delete kv.second;
        }
        cache_.clear();
    }
    cache_[cache_key] = m;
    compile_ms_ = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return m;
}

bool LensDevice::build(const std::string &lens_source, const LensBuildParams &p, uint32_t *cand, std::string *err) {
    kernel_ms_ = 0;
    Module *m = module_for(lens_source, false, err);
    if (!m) return false;
    Driver &d = driver();
    const size_t npix = static_cast<size_t>(p.width) * p.height;
    uint32_t *d_cand = nullptr;
    cudaError_t ce = cudaMalloc(&d_cand, npix * sizeof(uint32_t));
    if (ce != cudaSuccess) {
        *err = std::string("cudaMalloc: ") + cudaGetErrorString(ce);
        return false;
    }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    LensBuildParams params = p;
    void *args[] = {&params, &d_cand};
    const unsigned block = 128;
    cudaEventRecord(e0, nullptr);
    CUresult cr = d.LaunchKernel(m->fn, (p.width + block - 1) / block, static_cast<unsigned>(p.height), 1, block, 1, 1, 0, nullptr, args, nullptr);
    cudaEventRecord(e1, nullptr);
    bool ok = cr == CUDA_SUCCESS;
    if (!ok) *err = "cuLaunchKernel failed (CUresult " + std::to_string(static_cast<int>(cr)) + ")";
    if (ok) {
        ce = cudaMemcpy(cand, d_cand, npix * sizeof(uint32_t), cudaMemcpyDeviceToHost);  // synchronises
        if (ce != cudaSuccess) {
            *err = std::string("lens kernel: ") + cudaGetErrorString(ce);
            ok = false;
        } else {
            float ms = 0;
            cudaEventElapsedTime(&ms, e0, e1);
            kernel_ms_ = ms;
            ++launches_;
        }
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(d_cand);
    return ok;
}

bool LensDevice::forward_points(const std::string &lens_source, const LensBuildParams &p, std::vector<uint32_t> *undecided, std::string *err) {
    kernel_ms_ = 0;
    drop_forward_state();
    Module *m = module_for(lens_source, true, err);
    if (!m) return false;
    Driver &d = driver();
    const size_t n1 = static_cast<size_t>(p.platesize) + 1;
    const size_t npoints = static_cast<size_t>(p.numplates) * n1 * n1;
    if (npoints >= 0xFFFFFFFFull) {
        *err = "too many grid points";
        return false;
    }
    fwd_ = new ForwardState;
    fwd_->p = p;
    fwd_->npoints = npoints;
    cudaError_t ce = cudaMalloc(&fwd_->grid, npoints * sizeof(FwdPoint));
    if (ce == cudaSuccess) ce = cudaMalloc(&fwd_->status, npoints);
    if (ce == cudaSuccess) ce = cudaMalloc(&fwd_->undecided, kUndecidedCap * sizeof(unsigned));
    if (ce == cudaSuccess) ce = cudaMalloc(&fwd_->counters, 16 * sizeof(unsigned));
    if (ce == cudaSuccess) ce = cudaMemset(fwd_->counters, 0, 16 * sizeof(unsigned));
    if (ce != cudaSuccess) {
        *err = std::string("cudaMalloc: ") + cudaGetErrorString(ce);
        drop_forward_state();
        return false;
    }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    LensBuildParams params = p;
    unsigned cap = kUndecidedCap;
    void *args[] = {&params, &fwd_->grid, &fwd_->status, &fwd_->undecided, &fwd_->counters, &cap};
    const unsigned block = 128;
    cudaEventRecord(e0, nullptr);
    CUresult cr = d.LaunchKernel(m->fn, static_cast<unsigned>((n1 + block - 1) / block), static_cast<unsigned>(n1), static_cast<unsigned>(p.numplates), block, 1, 1, 0,
                                 nullptr, args, nullptr);
    cudaEventRecord(e1, nullptr);
    unsigned counters[16] = {};
    bool ok = cr == CUDA_SUCCESS;
    if (!ok) *err = "cuLaunchKernel failed (CUresult " + std::to_string(static_cast<int>(cr)) + ")";
    if (ok) {
        ce = cudaMemcpy(counters, fwd_->counters, sizeof counters, cudaMemcpyDeviceToHost);  // synchronises
        if (ce != cudaSuccess) {
            *err = std::string("lens kernel: ") + cudaGetErrorString(ce);
            ok = false;
        }
    }
    if (ok && counters[0] > kUndecidedCap) {
        *err = "too many grid points need the interpreter (" + std::to_string(counters[0]) + ")";
        ok = false;
    }
    if (ok) {
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        kernel_ms_ = ms;
        ++launches_;
        fwd_->nil_count = counters[1];
        undecided->resize(counters[0]);
        if (counters[0]) cudaMemcpy(undecided->data(), fwd_->undecided, counters[0] * sizeof(unsigned), cudaMemcpyDeviceToHost);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (!ok) drop_forward_state();
    return ok;
}

bool LensDevice::forward_finish(const std::vector<ForwardPatch> &patches, int32_t *idx, uint8_t *tint, int display[6],
                                std::vector<std::pair<uint32_t, int>> *messages, std::string *err) {
    if (!fwd_) {
        *err = "forward_finish without forward_points";
        return false;
    }
    const LensBuildParams &p = fwd_->p;
    const size_t npix = static_cast<size_t>(p.width) * p.height;
    ForwardPatch *d_patches = nullptr;
    unsigned *d_keys = nullptr;  // idxkey[npix] then tintkey[npix]
    FwdMessage *d_messages = nullptr;
    int32_t *d_idx = nullptr;
    uint8_t *d_tint = nullptr;
    cudaError_t ce = cudaMalloc(&d_keys, 2 * npix * sizeof(unsigned));
    if (ce == cudaSuccess) ce = cudaMemset(d_keys, 0, 2 * npix * sizeof(unsigned));
    if (ce == cudaSuccess) ce = cudaMalloc(&d_messages, kMessageCap * sizeof(FwdMessage));
    if (ce == cudaSuccess) ce = cudaMalloc(&d_idx, npix * sizeof(int32_t));
    if (ce == cudaSuccess) ce = cudaMalloc(&d_tint, npix);
    bool any_nil = fwd_->nil_count > 0;
    if (ce == cudaSuccess && !patches.empty()) {
        ce = cudaMalloc(&d_patches, patches.size() * sizeof(ForwardPatch));
        if (ce == cudaSuccess) ce = cudaMemcpy(d_patches, patches.data(), patches.size() * sizeof(ForwardPatch), cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) {
            const unsigned n = static_cast<unsigned>(patches.size());
            fwd_patch_kernel<<<(n + 255) / 256, 256>>>(fwd_->grid, fwd_->status, d_patches, n);
            ++launches_;
        }
        for (const ForwardPatch &pt : patches) any_nil = any_nil || pt.status != 1;
    }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    if (ce == cudaSuccess) {
        cudaEventRecord(e0, nullptr);
        if (any_nil) {
            const int threads = 2 * (p.platesize + 1);
            fwd_stale_kernel<<<(threads + 63) / 64, 64>>>(fwd_->grid, fwd_->status, p.platesize, p.numplates);
            ++launches_;
        }
        FwdGeom g;
        g.width = p.width;
        g.height = p.height;
        g.ps = p.platesize;
        g.numplates = p.numplates;
        g.rubix_block = p.rubix_block;
        g.rubix_pad = p.rubix_pad;
        g.rubix_unit_px = p.rubix_unit_px;
        memcpy(g.plates, p.plates, sizeof g.plates);
        FwdOut o{d_keys, d_keys + npix, fwd_->counters, d_messages};
        dim3 grid((p.platesize + 127) / 128, p.platesize, p.numplates);
        fwd_raster_kernel<<<grid, 128>>>(g, fwd_->grid, o);
        fwd_resolve_kernel<<<static_cast<unsigned>((npix + 255) / 256), 256>>>(d_keys, d_keys + npix, d_idx, d_tint, npix, p.platesize);
        launches_ += 2;
        cudaEventRecord(e1, nullptr);
        ce = cudaMemcpy(idx, d_idx, npix * sizeof(int32_t), cudaMemcpyDeviceToHost);
        if (ce == cudaSuccess) ce = cudaMemcpy(tint, d_tint, npix, cudaMemcpyDeviceToHost);
    }
    unsigned counters[16] = {};
    if (ce == cudaSuccess) ce = cudaMemcpy(counters, fwd_->counters, sizeof counters, cudaMemcpyDeviceToHost);
    bool ok = ce == cudaSuccess;
    if (!ok) *err = std::string("forward lensmap kernels: ") + cudaGetErrorString(ce);
    if (ok && counters[2] > kMessageCap) {
        *err = "too many 'maxdiff' messages to replay (" + std::to_string(counters[2]) + ")";
        ok = false;
    }
    if (ok) {
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        kernel_ms_ += ms;
        for (int i = 0; i < 6; ++i) display[i] = counters[3 + i] ? 1 : 0;
        std::vector<FwdMessage> msg(counters[2]);
        if (counters[2]) cudaMemcpy(msg.data(), d_messages, counters[2] * sizeof(FwdMessage), cudaMemcpyDeviceToHost);
        messages->clear();
        for (const FwdMessage &m : msg) messages->emplace_back(m.key, static_cast<int>(m.value));
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(d_patches);
    cudaFree(d_keys);
    cudaFree(d_messages);
    cudaFree(d_idx);
    cudaFree(d_tint);
    drop_forward_state();
    return ok;
}

}  // namespace blinky
