// C ABI of the H100 lens-warp path (include/blinky_b200.h): a thin veneer over
// FisheyeHost (host-side scripts/console/lensmap build) and WarpDevice (CUDA).
#include "../../include/blinky_b200.h"

#include <sched.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>
#include <stdexcept>
#include <string>

#include "fisheye_host.h"
#include "launch_plan.h"
#include "lens_device.h"
#include "lua_transpile.h"
#include "ray_texel.h"
#include "shard.h"
#include "tile_plan.h"
#include "tile_plan_device.h"
#include "warp_device.h"

using blinky::FisheyeHost;
using blinky::LensBuildParams;
using blinky::LensDevice;
using blinky::WarpDevice;

struct blinky_ctx {
    FisheyeHost host;
    std::unique_ptr<blinky::ShardGroup> shard;  // destroyed before the device it borrows
    std::unique_ptr<WarpDevice> dev;
    std::unique_ptr<LensDevice> lens_dev;
    std::string build_info;
    std::string err;
    std::string scratch;
    int layout_rowbytes = 0;              // blinky_set_face_layout: 0 = dense faces
    std::vector<int32_t> layout_origins;  // (x, y) per plate
    bool device_plan = false;             // the resident tile plan was made on the GPU (blinky_set_lensmap_device)
};

namespace {

int set_err(blinky_ctx *c, int code, const std::string &msg) {
    c->err = msg;
    return code;
}

// CPUs this process may really use: the affinity mask, capped by the cgroup CPU quota
// (a container can see 128 cores and be allowed 24)
int usable_cpus() {
    int n = static_cast<int>(std::thread::hardware_concurrency());
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) n = CPU_COUNT(&set);
    FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
    if (f) {
        char quota[64];
        long period = 0;
        if (fscanf(f, "%63s %ld", quota, &period) == 2 && strcmp(quota, "max") != 0 && period > 0) {
            int q = static_cast<int>((atol(quota) + period - 1) / period);
            if (q >= 1 && q < n) n = q;
        }
        fclose(f);
    }
    return n < 1 ? 1 : n;
}

// The tile plan of the current lensmap, classified on `threads` host threads.  TMA needs 16-byte aligned plate rows;
// other plate sizes get GATHER tiles only.
blinky::TilePlan current_plan(blinky_ctx *c, int threads) {
    return blinky::make_tile_plan(c->host.packed().data(), c->host.width(), c->host.height(), c->host.platesize(), c->host.platesize() % 16 == 0,
                                  threads);
}

// A map planned on the GPU stays there until a host-side query needs it; then it is copied back once and kept.
bool host_map(blinky_ctx *c) {
    if (c->host.map_on_host()) return true;
    std::vector<uint32_t> m(static_cast<size_t>(c->host.width()) * c->host.height());
    if (!c->dev->download_lensmap(m.data())) {
        c->err = c->dev->last_error();
        return false;
    }
    c->host.fill_lensmap(std::move(m));
    return true;
}

// the plates' palette LUTs, as the device keeps them
void plate_luts(blinky_ctx *c, uint8_t out[BLINKY_MAX_PLATES * 256]) {
    for (int i = 0; i < BLINKY_MAX_PLATES; ++i) memcpy(out + i * 256, c->host.plate(i).palette, 256);
}

// Installs the current lensmap on the device: the host's map, planned and staged here, or (device != null) a map and
// plan the GPU planner left in device memory.
bool upload(blinky_ctx *c, blinky::DevicePlan *device = nullptr) {
    if (!c->dev || !c->host.built()) return true;
    blinky::DevicePlan staged;
    if (!device) {
        if (!host_map(c)) return false;
        const size_t npix = static_cast<size_t>(c->host.width()) * c->host.height();
        if (blinky::stage_lensmap_host(c->dev->device(), c->host.packed().data(), npix, WarpDevice::padded_pixels(npix),
                                       current_plan(c, c->host.worker_threads()), &staged, &c->err) != BLINKY_OK)
            return false;
    }
    blinky::LensmapUpload lm;
    lm.width = c->host.width();
    lm.height = c->host.height();
    lm.platesize = c->host.platesize();
    lm.numplates = c->host.map_numplates();
    for (int i = 0; i < BLINKY_MAX_PLATES; ++i) {
        lm.display[i] = i < c->host.map_numplates() ? c->host.plate(i).display : 0;
        memcpy(lm.plate_rect[i], c->host.plate_rect(i), sizeof lm.plate_rect[i]);
    }
    uint8_t luts[BLINKY_MAX_PLATES * 256];
    plate_luts(c, luts);
    lm.palmaps = luts;
    lm.rubix = c->host.rubix_enabled();
    lm.span_off = c->host.row_span_offsets().data();
    lm.spans = c->host.row_spans().data();
    lm.nspans = c->host.row_spans().size() / 2;
    c->device_plan = device != nullptr;
    if (!c->dev->install(lm, std::move(device ? *device : staged))) {
        c->err = c->dev->last_error();
        return false;
    }
    return true;
}

}  // namespace

extern "C" {

int blinky_create(int device, blinky_ctx **out) {
    if (!out) return BLINKY_E_INVALID;
    *out = nullptr;
    blinky_ctx *c;
    try {
        c = new blinky_ctx();
    } catch (std::exception &) {
        return BLINKY_E_NOMEM;
    }
    c->host.set_worker_threads(usable_cpus());
    if (device >= 0) {
        try {
            c->dev.reset(new WarpDevice(device));
            c->lens_dev.reset(new LensDevice(device));
            c->host.set_device_builder(c->lens_dev.get());
        } catch (std::exception &e) {
            // no silent CPU fallback: hand back a context that explains itself
            c->err = e.what();
            *out = c;
            return BLINKY_E_CUDA;
        }
    }
    *out = c;
    return BLINKY_OK;
}

void blinky_destroy(blinky_ctx *ctx) { delete ctx; }

const char *blinky_last_error(blinky_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
const char *blinky_version(void) { return "blinky_b200 0.1 (sm_90a)"; }

void blinky_set_print_callback(blinky_ctx *ctx, blinky_print_fn fn, void *user) { ctx->host.set_print(fn, user); }
void blinky_set_exec_callback(blinky_ctx *ctx, blinky_exec_fn fn, void *user) { ctx->host.set_exec(fn, user); }
const char *blinky_log(blinky_ctx *ctx) { return ctx->host.log().c_str(); }
void blinky_log_clear(blinky_ctx *ctx) { ctx->host.clear_log(); }

int blinky_set_basedir(blinky_ctx *ctx, const char *basedir) {
    if (!basedir) return set_err(ctx, BLINKY_E_INVALID, "basedir is NULL");
    ctx->host.set_basedir(basedir);
    return BLINKY_OK;
}

int blinky_set_palette(blinky_ctx *ctx, const uint8_t palette[768]) {
    if (!palette) return set_err(ctx, BLINKY_E_INVALID, "palette is NULL");
    ctx->host.set_palette(palette);
    if (!ctx->dev || !ctx->host.built()) return BLINKY_OK;
    uint8_t luts[BLINKY_MAX_PLATES * 256];
    plate_luts(ctx, luts);
    return ctx->dev->set_luts(luts) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

int blinky_command(blinky_ctx *ctx, const char *text) {
    if (!text) return set_err(ctx, BLINKY_E_INVALID, "command is NULL");
    if (!ctx->host.command(text)) return set_err(ctx, BLINKY_E_INVALID, std::string("unknown command: ") + text);
    if (ctx->dev) ctx->dev->set_rubix(ctx->host.rubix_enabled());
    return BLINKY_OK;
}

int blinky_load_globe(blinky_ctx *ctx, const char *name) {
    if (!name) return set_err(ctx, BLINKY_E_INVALID, "name is NULL");
    return ctx->host.cmd_globe(name, nullptr) ? BLINKY_OK : set_err(ctx, BLINKY_E_SCRIPT, "not a valid globe");
}
int blinky_load_lens(blinky_ctx *ctx, const char *name) {
    if (!name) return set_err(ctx, BLINKY_E_INVALID, "name is NULL");
    return ctx->host.cmd_lens(name, nullptr) ? BLINKY_OK : set_err(ctx, BLINKY_E_SCRIPT, "not a valid lens");
}
int blinky_load_globe_source(blinky_ctx *ctx, const char *name, const char *src) {
    if (!name || !src) return set_err(ctx, BLINKY_E_INVALID, "name/source is NULL");
    std::string s(src);
    return ctx->host.cmd_globe(name, &s) ? BLINKY_OK : set_err(ctx, BLINKY_E_SCRIPT, "not a valid globe");
}
int blinky_load_lens_source(blinky_ctx *ctx, const char *name, const char *src) {
    if (!name || !src) return set_err(ctx, BLINKY_E_INVALID, "name/source is NULL");
    std::string s(src);
    return ctx->host.cmd_lens(name, &s) ? BLINKY_OK : set_err(ctx, BLINKY_E_SCRIPT, "not a valid lens");
}

int blinky_set_zoom(blinky_ctx *ctx, int zoom_type, int fov) {
    if (zoom_type < BLINKY_ZOOM_NONE || zoom_type > BLINKY_ZOOM_CONTAIN) return set_err(ctx, BLINKY_E_INVALID, "bad zoom type");
    ctx->host.set_zoom(zoom_type, fov);
    return BLINKY_OK;
}
int blinky_set_rubix(blinky_ctx *ctx, int enabled) {
    ctx->host.set_rubix(enabled != 0);
    if (ctx->dev) ctx->dev->set_rubix(enabled != 0);
    return BLINKY_OK;
}
int blinky_set_rubixgrid(blinky_ctx *ctx, int numcells, double cell, double pad) {
    ctx->host.set_rubixgrid(numcells, cell, pad);
    return BLINKY_OK;
}

int blinky_build_lensmap(blinky_ctx *ctx, int width, int height, int platesize, int threads) {
    if (width <= 0 || height <= 0) return set_err(ctx, BLINKY_E_INVALID, "width/height must be positive");
    if (threads < 0) threads = usable_cpus();
    int rc = ctx->host.build_lensmap(width, height, platesize, threads);
    ctx->build_info = ctx->host.build_info();
    if (ctx->lens_dev && ctx->build_info.compare(0, 6, "device") == 0) {
        char t[96];
        snprintf(t, sizeof t, " (NVRTC %.0f ms, kernel %.3f ms)", ctx->lens_dev->last_compile_ms(), ctx->lens_dev->last_kernel_ms());
        ctx->build_info += t;
    }
    // the (possibly empty) map is published even on failure, as the reference renders it
    auto t0 = std::chrono::steady_clock::now();
    const bool uploaded = upload(ctx);
    if (ctx->dev) {
        char t[64];
        snprintf(t, sizeof t, ", plan+upload %.1f ms", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
        ctx->build_info += t;
    }
    if (!uploaded) return BLINKY_E_CUDA;
    switch (rc) {
        case 0: return BLINKY_OK;
        case -1: return set_err(ctx, BLINKY_E_INVALID, "bad size (platesize too large for the 28-bit texel index?)");
        case -3: return set_err(ctx, BLINKY_E_ZOOM, "zoom could not be computed for this lens: " + ctx->host.log());
        case -7: return set_err(ctx, BLINKY_E_STATE, "lens or globe is not valid");
        default: return set_err(ctx, BLINKY_E_SCRIPT, "lens script failed during the build: " + ctx->host.log());
    }
}

int blinky_set_lensmap(blinky_ctx *ctx, int width, int height, int platesize, int numplates, const uint32_t *packed) {
    std::string why;
    auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point t) {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
    };
    if (!ctx->host.set_lensmap(width, height, platesize, numplates, packed, &why)) return set_err(ctx, BLINKY_E_INVALID, "blinky_set_lensmap: " + why);
    char t[128];
    snprintf(t, sizeof t, "supplied (host memory); finish %.1f ms", ms_since(t0));
    ctx->build_info = t;
    t0 = std::chrono::steady_clock::now();
    const bool uploaded = upload(ctx);
    if (ctx->dev) {
        snprintf(t, sizeof t, ", plan+upload %.1f ms", ms_since(t0));
        ctx->build_info += t;
    }
    return uploaded ? BLINKY_OK : BLINKY_E_CUDA;
}

}  // extern "C"

namespace {

// blinky_set_raymap and the host path of blinky_set_raymap_device: sizes checked, rays in host memory
int set_raymap_host(blinky_ctx *ctx, const char *who, int width, int height, int platesize, const float *rays, const std::string &path) {
    auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point t) {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
    };
    if (ctx->host.set_raymap(width, height, platesize, rays) != 0)
        return set_err(ctx, BLINKY_E_SCRIPT, std::string(who) + ": globe_plate failed: " + ctx->host.log());
    char t[96];
    snprintf(t, sizeof t, "; map %.1f ms", ms_since(t0));
    ctx->build_info = "ray map, " + path + t;
    t0 = std::chrono::steady_clock::now();
    const bool uploaded = upload(ctx);
    if (ctx->dev) {
        snprintf(t, sizeof t, ", plan+upload %.1f ms", ms_since(t0));
        ctx->build_info += t;
    }
    return uploaded ? BLINKY_OK : BLINKY_E_CUDA;
}

// the checks both ray-map entry points make before anything changes
int check_raymap(blinky_ctx *ctx, const char *who, int width, int height, int *platesize, const float *rays) {
    if (!rays || reinterpret_cast<uintptr_t>(rays) % 4 != 0) return set_err(ctx, BLINKY_E_INVALID, std::string(who) + ": rays must be a non-NULL, 4-byte aligned pointer");
    std::string why;
    const int rc = ctx->host.check_raymap(width, height, platesize, &why);
    if (rc != 0) return set_err(ctx, rc == -7 ? BLINKY_E_STATE : BLINKY_E_INVALID, std::string(who) + ": " + why);
    return BLINKY_OK;
}

// the checks both ray-export entry points make before anything runs; *scale: the zoom of a width x height build
int check_export(blinky_ctx *ctx, const char *who, int width, int height, const float *rays, double *scale) {
    if (!rays || reinterpret_cast<uintptr_t>(rays) % 4 != 0) return set_err(ctx, BLINKY_E_INVALID, std::string(who) + ": rays must be a non-NULL, 4-byte aligned pointer");
    if (width <= 0 || height <= 0) return set_err(ctx, BLINKY_E_INVALID, std::string(who) + ": width and height must be positive");
    std::string why;
    const int rc = ctx->host.check_rays(width, height, scale, &why);
    if (rc == -7) return set_err(ctx, BLINKY_E_STATE, std::string(who) + ": " + why);
    if (rc != 0) return set_err(ctx, BLINKY_E_ZOOM, std::string(who) + ": zoom could not be computed for this lens: " + ctx->host.log());
    return BLINKY_OK;
}

// blinky_get_raymap and the host path of blinky_get_raymap_device: the rays into host memory on the worker threads
int get_raymap_host(blinky_ctx *ctx, const char *who, int width, int height, double scale, float *rays, const std::string &path) {
    auto t0 = std::chrono::steady_clock::now();
    if (ctx->host.export_rays(width, height, scale, rays) != 0)
        return set_err(ctx, BLINKY_E_SCRIPT, std::string(who) + ": lens_inverse failed: " + ctx->host.log());
    char t[64];
    snprintf(t, sizeof t, "; rays %.1f ms", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    ctx->build_info = "ray export, " + path + t;
    return BLINKY_OK;
}

// the checks both forward ray-export entry points make before anything runs; *platesize: the build's, *scale: its zoom
int check_export_forward(blinky_ctx *ctx, const char *who, int width, int height, int *platesize, const float *rays, double *scale) {
    if (!rays || reinterpret_cast<uintptr_t>(rays) % 4 != 0) return set_err(ctx, BLINKY_E_INVALID, std::string(who) + ": rays must be a non-NULL, 4-byte aligned pointer");
    if (width <= 0 || height <= 0) return set_err(ctx, BLINKY_E_INVALID, std::string(who) + ": width and height must be positive");
    std::string why;
    const int rc = ctx->host.check_rays_forward(width, height, platesize, scale, &why);
    if (rc == -1) return set_err(ctx, BLINKY_E_INVALID, std::string(who) + ": " + why);
    if (rc == -7) return set_err(ctx, BLINKY_E_STATE, std::string(who) + ": " + why);
    if (rc != 0) return set_err(ctx, BLINKY_E_ZOOM, std::string(who) + ": zoom could not be computed for this lens: " + ctx->host.log());
    return BLINKY_OK;
}

// blinky_get_raymap_forward and the host path of blinky_get_raymap_forward_device: the serial forward builder into host memory
int get_raymap_forward_host(blinky_ctx *ctx, const char *who, int width, int height, int platesize, double scale, float *rays, const std::string &path) {
    auto t0 = std::chrono::steady_clock::now();
    if (ctx->host.export_rays_forward(width, height, platesize, scale, rays) != 0)
        return set_err(ctx, BLINKY_E_SCRIPT, std::string(who) + ": lens_forward failed: " + ctx->host.log());
    char t[64];
    snprintf(t, sizeof t, "; rays %.1f ms", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    ctx->build_info = "ray export (forward), " + path + t;
    return BLINKY_OK;
}

}  // namespace

extern "C" {

int blinky_set_raymap(blinky_ctx *ctx, int width, int height, int platesize, const float *rays) {
    const char *who = "blinky_set_raymap";
    const int rc = check_raymap(ctx, who, width, height, &platesize, rays);
    return rc != BLINKY_OK ? rc : set_raymap_host(ctx, who, width, height, platesize, rays, "host");
}

int blinky_get_raymap(blinky_ctx *ctx, int width, int height, float *rays) {
    const char *who = "blinky_get_raymap";
    double scale;
    const int rc = check_export(ctx, who, width, height, rays, &scale);
    return rc != BLINKY_OK ? rc : get_raymap_host(ctx, who, width, height, scale, rays, "host");
}

int blinky_get_raymap_forward(blinky_ctx *ctx, int width, int height, int platesize, float *rays) {
    const char *who = "blinky_get_raymap_forward";
    double scale;
    const int rc = check_export_forward(ctx, who, width, height, &platesize, rays, &scale);
    return rc != BLINKY_OK ? rc : get_raymap_forward_host(ctx, who, width, height, platesize, scale, rays, "host");
}

const char *blinky_build_info(blinky_ctx *ctx) { return ctx->build_info.c_str(); }

int blinky_compile_lens(blinky_ctx *ctx, int forward, size_t *cubin_bytes) {
    std::string src, why;
    if (!ctx->host.lens_device_source(true, &src, &why, forward != 0, true)) return set_err(ctx, BLINKY_E_SCRIPT, why);
    std::vector<char> cubin;
    std::string log;
    if (!LensDevice::compile(src, forward != 0, &cubin, &log)) return set_err(ctx, BLINKY_E_CUDA, log);
    if (cubin_bytes) *cubin_bytes = cubin.size();
    return BLINKY_OK;
}

int blinky_probe_math(blinky_ctx *ctx, int op, const double *d_a, const double *d_b, double *d_v, double *d_e, size_t n, void *stream) {
    const bool binary = op == BLINKY_PROBE_ATAN2 || op == BLINKY_PROBE_LOGB || op == BLINKY_PROBE_POW || op == BLINKY_PROBE_FMOD ||
                        op == BLINKY_PROBE_DIV;
    if (op < 0 || op >= BLINKY_PROBE_COUNT) return set_err(ctx, BLINKY_E_INVALID, "blinky_probe_math: unknown op");
    const std::string prelude = blinky::transpile_prelude(true, false);
    if (n == 0) {
        std::vector<char> cubin;
        std::string log;
        return LensDevice::compile_unit(prelude + LensDevice::probe_tail(), &cubin, &log) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, log);
    }
    if (!ctx->lens_dev) return set_err(ctx, BLINKY_E_NODEVICE, "blinky_probe_math: this context has no GPU");
    for (const void *p : {static_cast<const void *>(d_a), static_cast<const void *>(d_v), static_cast<const void *>(d_e),
                          binary ? static_cast<const void *>(d_b) : static_cast<const void *>(d_a)})
        if (!p || reinterpret_cast<uintptr_t>(p) % 8 != 0)
            return set_err(ctx, BLINKY_E_INVALID, "blinky_probe_math: arguments and results must be non-NULL, 8-byte aligned pointers");
    if (LensDevice::capturing(stream)) return set_err(ctx, BLINKY_E_STATE, "blinky_probe_math: the stream is capturing a graph");
    std::string why;
    return ctx->lens_dev->probe_math(prelude, op, d_a, d_b, d_v, d_e, n, stream, &why) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, why);
}

int blinky_needs_rebuild(blinky_ctx *ctx, int w, int h, int ps) { return ctx->host.needs_rebuild(w, h, ps) ? 1 : 0; }

int blinky_fisheye_enabled(blinky_ctx *ctx) { return ctx->host.fisheye_enabled() ? 1 : 0; }
int blinky_lens_valid(blinky_ctx *ctx) { return ctx->host.lens_valid() ? 1 : 0; }
int blinky_globe_valid(blinky_ctx *ctx) { return ctx->host.globe_valid() ? 1 : 0; }
const char *blinky_lens_name(blinky_ctx *ctx) { return ctx->host.lens_name().c_str(); }
const char *blinky_globe_name(blinky_ctx *ctx) { return ctx->host.globe_name().c_str(); }
const char *blinky_lens_onload(blinky_ctx *ctx) { return ctx->host.onload().c_str(); }
int blinky_map_type(blinky_ctx *ctx) { return ctx->host.map_type(); }
int blinky_zoom_type(blinky_ctx *ctx) { return ctx->host.zoom_type(); }
int blinky_zoom_fov(blinky_ctx *ctx) { return ctx->host.zoom_fov(); }
int blinky_max_fov(blinky_ctx *ctx) { return ctx->host.max_fov(); }
int blinky_max_vfov(blinky_ctx *ctx) { return ctx->host.max_vfov(); }
double blinky_lens_width(blinky_ctx *ctx) { return ctx->host.lens_width(); }
double blinky_lens_height(blinky_ctx *ctx) { return ctx->host.lens_height(); }
double blinky_scale(blinky_ctx *ctx) { return ctx->host.scale(); }
int blinky_rubix_enabled(blinky_ctx *ctx) { return ctx->host.rubix_enabled() ? 1 : 0; }
int blinky_numplates(blinky_ctx *ctx) { return ctx->host.numplates(); }
int blinky_platesize(blinky_ctx *ctx) { return ctx->host.platesize(); }
int blinky_width(blinky_ctx *ctx) { return ctx->host.width(); }
int blinky_height(blinky_ctx *ctx) { return ctx->host.height(); }

int blinky_get_plates(blinky_ctx *ctx, float *out, int max_plates) {
    int n = ctx->host.numplates();
    for (int i = 0; i < n && i < max_plates; ++i) {
        const blinky::Plate &p = ctx->host.plate(i);
        float *o = out + i * 11;
        memcpy(o, p.forward, 12);
        memcpy(o + 3, p.right, 12);
        memcpy(o + 6, p.up, 12);
        o[9] = p.fov;
        o[10] = p.dist;
    }
    return n;
}

int blinky_get_display(blinky_ctx *ctx, int out[BLINKY_MAX_PLATES]) {
    const int n = ctx->host.built() ? ctx->host.map_numplates() : ctx->host.numplates();
    for (int i = 0; i < BLINKY_MAX_PLATES; ++i) out[i] = i < n ? ctx->host.plate(i).display : 0;
    return BLINKY_OK;
}

double blinky_plate_fov(blinky_ctx *ctx, int plate) {
    if (plate < 0 || plate >= ctx->host.numplates()) return 0;
    return ctx->host.plate(plate).fov;
}

int blinky_get_palmaps(blinky_ctx *ctx, uint8_t out[BLINKY_MAX_PLATES * 256]) {
    for (int i = 0; i < BLINKY_MAX_PLATES; ++i) memcpy(out + i * 256, ctx->host.plate(i).palette, 256);
    return BLINKY_OK;
}

int blinky_get_lensmap(blinky_ctx *ctx, int32_t *idx, uint8_t *tint) {
    if (!ctx->host.built()) return set_err(ctx, BLINKY_E_STATE, "no lensmap built");
    if (!host_map(ctx)) return BLINKY_E_CUDA;
    if (idx) memcpy(idx, ctx->host.indices().data(), ctx->host.indices().size() * sizeof(int32_t));
    if (tint) memcpy(tint, ctx->host.tints().data(), ctx->host.tints().size());
    return BLINKY_OK;
}

int blinky_get_lensmap_packed(blinky_ctx *ctx, uint32_t *out) {
    if (!ctx->host.built()) return set_err(ctx, BLINKY_E_STATE, "no lensmap built");
    if (!host_map(ctx)) return BLINKY_E_CUDA;
    memcpy(out, ctx->host.packed().data(), ctx->host.packed().size() * sizeof(uint32_t));
    return BLINKY_OK;
}

int64_t blinky_mapped_pixels(blinky_ctx *ctx) { return ctx->host.mapped_pixels(); }

int blinky_lens_inverse(blinky_ctx *ctx, double x, double y, double ray_out[3]) { return ctx->host.lens_inverse(x, y, ray_out); }
int blinky_lens_forward(blinky_ctx *ctx, double rx, double ry, double rz, double *x, double *y) {
    return ctx->host.lens_forward(rx, ry, rz, x, y);
}

int blinky_globe_plate(blinky_ctx *ctx, double x, double y, double z, int *plate) {
    int p = -1;
    const int rc = ctx->host.globe_plate(x, y, z, &p);
    if (plate) *plate = p;
    return rc;
}

int blinky_lens_source(blinky_ctx *ctx, int flavour, char *buf, size_t bufsize) {
    std::string s, why;
    if (flavour & 32) {
        if (!ctx->host.lens_device_source((flavour & 1) != 0, &s, &why)) return set_err(ctx, BLINKY_E_SCRIPT, why);
        s += LensDevice::rays_tail();
    } else if (flavour & 16) {
        if (!ctx->host.raymap_device_source((flavour & 1) != 0, &s, &why)) return set_err(ctx, BLINKY_E_SCRIPT, why);
        s += LensDevice::raymap_tail(blinky::source_has_globe_plate(s));
    } else if (flavour & 8) {
        if (!ctx->host.globe_plate_device_source((flavour & 1) != 0, &s, &why)) return set_err(ctx, BLINKY_E_SCRIPT, why);
    } else {
        // with the kernel: the unit NVRTC compiles, i.e. with the globe's globe_plate when it has one
        const bool kernel = (flavour & 4) != 0;
        if (!ctx->host.lens_device_source((flavour & 1) != 0, &s, &why, (flavour & 2) != 0, kernel)) return set_err(ctx, BLINKY_E_SCRIPT, why);
        if (kernel) s += LensDevice::kernel_tail((flavour & 2) != 0, blinky::source_has_globe_plate(s));
    }
    if (buf && bufsize) {
        size_t n = s.size() < bufsize - 1 ? s.size() : bufsize - 1;
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return static_cast<int>(s.size());
}

int blinky_write_config(blinky_ctx *ctx, char *buf, size_t bufsize) {
    std::string s = ctx->host.write_config();
    if (buf && bufsize) {
        size_t n = s.size() < bufsize - 1 ? s.size() : bufsize - 1;
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return static_cast<int>(s.size());
}

int blinky_set_face_layout(blinky_ctx *ctx, int rowbytes, const int32_t *origins, int nplates) {
    if (rowbytes < 0) return set_err(ctx, BLINKY_E_INVALID, "blinky_set_face_layout: rowbytes < 0");
    if (rowbytes > 0) {
        if (!origins) return set_err(ctx, BLINKY_E_INVALID, "blinky_set_face_layout: origins is NULL");
        if (nplates < 1 || nplates > BLINKY_MAX_PLATES) return set_err(ctx, BLINKY_E_INVALID, "blinky_set_face_layout: nplates must be 1..6");
        for (int i = 0; i < 2 * nplates; ++i)
            if (origins[i] < 0) return set_err(ctx, BLINKY_E_INVALID, "blinky_set_face_layout: negative plate origin");
        ctx->layout_origins.assign(origins, origins + 2 * nplates);
    } else {
        ctx->layout_origins.clear();
    }
    ctx->layout_rowbytes = rowbytes;
    if (ctx->dev) ctx->dev->set_face_layout(rowbytes, ctx->layout_origins.data(), static_cast<int>(ctx->layout_origins.size() / 2));
    return BLINKY_OK;
}

int blinky_saveglobe_pending(blinky_ctx *ctx) { return ctx->host.saveglobe_pending() ? 1 : 0; }
int blinky_save_globe(blinky_ctx *ctx, const uint8_t *faces_host, const char *directory) {
    if (!faces_host) return set_err(ctx, BLINKY_E_INVALID, "faces is NULL");
    if (!ctx->host.built()) return set_err(ctx, BLINKY_E_STATE, "no lensmap built (plate size unknown)");
    if (ctx->layout_rowbytes > 0) {
        // every plate is written: each needs an origin that fits the row pitch
        const int ps = ctx->host.platesize(), n = static_cast<int>(ctx->layout_origins.size() / 2);
        if (ctx->host.numplates() > n) return set_err(ctx, BLINKY_E_INVALID, "blinky_save_globe: the face layout has no origin for every plate");
        for (int i = 0; i < n; ++i)
            if (static_cast<int64_t>(ctx->layout_origins[2 * i]) + ps > ctx->layout_rowbytes)
                return set_err(ctx, BLINKY_E_INVALID, "blinky_save_globe: a plate of the face layout does not fit its rowbytes");
    }
    return ctx->host.save_globe(faces_host, directory ? directory : "", ctx->layout_rowbytes, ctx->layout_origins.data())
               ? BLINKY_OK
               : set_err(ctx, BLINKY_E_INVALID, "could not write a PCX file");
}

// ---- GPU-only entry points: no CPU fallback, fail loudly ------------------

#define NEED_DEVICE(ctx)                                                                                              \
    if (!(ctx)->dev)                                                                                                  \
        return set_err(ctx, BLINKY_E_NODEVICE,                                                                        \
                       "this context has no GPU; the warp runs only as sm_90a CUDA kernels (no CPU fallback)")

int blinky_set_kernel(blinky_ctx *ctx, int variant) {
    NEED_DEVICE(ctx);
    if (variant != BLINKY_KERNEL_AUTO && variant != BLINKY_KERNEL_GATHER && variant != BLINKY_KERNEL_TMA)
        return set_err(ctx, BLINKY_E_INVALID, "blinky_set_kernel: unknown kernel variant");
    ctx->dev->set_kernel(variant);
    return BLINKY_OK;
}

int blinky_set_lensmap_device(blinky_ctx *ctx, int width, int height, int platesize, int numplates, const uint32_t *d_packed, void *stream) {
    NEED_DEVICE(ctx);
    std::string why;
    if (!FisheyeHost::check_lensmap_size(width, height, platesize, numplates, &why)) return set_err(ctx, BLINKY_E_INVALID, "blinky_set_lensmap_device: " + why);
    if (!d_packed) return set_err(ctx, BLINKY_E_INVALID, "blinky_set_lensmap_device: map is NULL");
    auto t0 = std::chrono::steady_clock::now();
    blinky::DevicePlan dp;
    const int rc = blinky::plan_lensmap_device(ctx->dev->device(), d_packed, width, height, platesize, numplates,
                                               WarpDevice::padded_pixels(static_cast<size_t>(width) * height), stream, &dp, &why);
    if (rc != BLINKY_OK) return set_err(ctx, rc, why);
    const double ms_plan = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    t0 = std::chrono::steady_clock::now();
    ctx->host.adopt_lensmap(width, height, platesize, numplates, dp.display, dp.rect, dp.mapped, std::move(dp.span_off), std::move(dp.spans));
    if (!upload(ctx, &dp)) return BLINKY_E_CUDA;
    char t[128];
    snprintf(t, sizeof t, "supplied (device memory); plan %.3f ms, adopt %.3f ms", ms_plan,
             std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    ctx->build_info = t;
    return BLINKY_OK;
}

int blinky_set_raymap_device(blinky_ctx *ctx, int width, int height, int platesize, const float *d_rays, void *stream) {
    NEED_DEVICE(ctx);
    const char *who = "blinky_set_raymap_device";
    int rc = check_raymap(ctx, who, width, height, &platesize, d_rays);
    if (rc != BLINKY_OK) return rc;
    auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point t) {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
    };
    const size_t npix = static_cast<size_t>(width) * height;
    std::string why;
    uint32_t *d_map = nullptr;
    size_t settled = 0;
    rc = ctx->host.raymap_device(width, height, platesize, d_rays, stream, &d_map, &settled, &why);
    if (rc == -2) return set_err(ctx, BLINKY_E_SCRIPT, std::string(who) + ": globe_plate failed: " + ctx->host.log());
    if (rc == 1) {
        std::vector<float> rays(3 * npix);
        if (!ctx->lens_dev->copy_to_host(rays.data(), d_rays, rays.size() * sizeof(float), stream, &ctx->err)) return BLINKY_E_CUDA;
        return set_raymap_host(ctx, who, width, height, platesize, rays.data(), "host (" + why + ")");
    }
    const double ms_map = ms_since(t0);
    t0 = std::chrono::steady_clock::now();
    // entries on the stale slots of a globe_plate may index any of the six plates, as in a build's map
    blinky::DevicePlan dp;
    rc = blinky::plan_lensmap_device(ctx->dev->device(), d_map, width, height, platesize, BLINKY_MAX_PLATES, WarpDevice::padded_pixels(npix), stream,
                                     &dp, &why);
    if (rc != BLINKY_OK) return set_err(ctx, rc, why);
    ctx->host.adopt_lensmap(width, height, platesize, ctx->host.numplates(), dp.display, dp.rect, dp.mapped, std::move(dp.span_off), std::move(dp.spans));
    if (!upload(ctx, &dp)) return BLINKY_E_CUDA;
    char t[256];
    snprintf(t, sizeof t, "ray map, device: %zu of %zu pixels settled by the interpreter; map %.3f ms (NVRTC %.0f ms, kernel %.3f ms), plan+adopt %.3f ms",
             settled, npix, ms_map, ctx->lens_dev->last_compile_ms(), ctx->lens_dev->last_kernel_ms(), ms_since(t0));
    ctx->build_info = t;
    return BLINKY_OK;
}

int blinky_get_raymap_device(blinky_ctx *ctx, int width, int height, float *d_rays, void *stream) {
    NEED_DEVICE(ctx);
    const char *who = "blinky_get_raymap_device";
    double scale;
    int rc = check_export(ctx, who, width, height, d_rays, &scale);
    if (rc != BLINKY_OK) return rc;
    // the host settles flagged pixels and the call returns with the field complete: nothing here can be captured
    if (LensDevice::capturing(stream)) return set_err(ctx, BLINKY_E_STATE, std::string(who) + ": the stream is capturing a graph");
    const size_t npix = static_cast<size_t>(width) * height;
    std::string why;
    size_t settled = 0;
    rc = ctx->host.export_rays_device(width, height, scale, d_rays, stream, &settled, &why);
    if (rc == -2) return set_err(ctx, BLINKY_E_SCRIPT, std::string(who) + ": lens_inverse failed: " + ctx->host.log());
    if (rc == 1) {
        std::vector<float> rays(3 * npix);
        rc = get_raymap_host(ctx, who, width, height, scale, rays.data(), "host (" + why + ")");
        if (rc != BLINKY_OK) return rc;
        return ctx->lens_dev->copy_to_device(d_rays, rays.data(), rays.size() * sizeof(float), stream, &ctx->err) ? BLINKY_OK : BLINKY_E_CUDA;
    }
    char t[192];
    snprintf(t, sizeof t, "ray export, device: %zu of %zu pixels settled by the interpreter; NVRTC %.0f ms, kernel %.3f ms", settled, npix,
             ctx->lens_dev->last_compile_ms(), ctx->lens_dev->last_kernel_ms());
    ctx->build_info = t;
    return BLINKY_OK;
}

int blinky_get_raymap_forward_device(blinky_ctx *ctx, int width, int height, int platesize, float *d_rays, void *stream) {
    NEED_DEVICE(ctx);
    const char *who = "blinky_get_raymap_forward_device";
    double scale;
    int rc = check_export_forward(ctx, who, width, height, &platesize, d_rays, &scale);
    if (rc != BLINKY_OK) return rc;
    // the host settles grid points between the kernels and the call returns with the field complete: nothing here can be captured
    if (LensDevice::capturing(stream)) return set_err(ctx, BLINKY_E_STATE, std::string(who) + ": the stream is capturing a graph");
    const size_t npix = static_cast<size_t>(width) * height;
    std::string why;
    size_t settled = 0;
    rc = ctx->host.export_rays_forward_device(width, height, platesize, scale, d_rays, stream, &settled, &why);
    if (rc == -2) return set_err(ctx, BLINKY_E_SCRIPT, std::string(who) + ": lens_forward failed: " + ctx->host.log());
    if (rc == 1) {
        std::vector<float> rays(3 * npix);
        rc = get_raymap_forward_host(ctx, who, width, height, platesize, scale, rays.data(), "host (" + why + ")");
        if (rc != BLINKY_OK) return rc;
        return ctx->lens_dev->copy_to_device(d_rays, rays.data(), rays.size() * sizeof(float), stream, &ctx->err) ? BLINKY_OK : BLINKY_E_CUDA;
    }
    char t[256];
    snprintf(t, sizeof t, "ray export (forward), device: %zu grid points settled by the interpreter; NVRTC %.0f ms, kernels %.3f ms (rays %.3f ms)",
             settled, ctx->lens_dev->last_compile_ms(), ctx->lens_dev->last_kernel_ms(), ctx->lens_dev->last_ray_kernel_ms());
    ctx->build_info = t;
    return BLINKY_OK;
}

int blinky_set_background(blinky_ctx *ctx, const uint8_t *bg) {
    NEED_DEVICE(ctx);
    return ctx->dev->set_background(bg) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

}  // extern "C"

namespace {

blinky::GlobeState globe_state(blinky_ctx *ctx) {
    blinky::GlobeState g;
    g.valid = ctx->host.globe_valid();
    g.plate_script = ctx->host.has_globe_plate();
    g.plates = ctx->host.numplates();
    return g;
}

// The view entry points: r into the view rectangle at (x0, y0) of screens whose rows are rowbytes bytes apart, from
// the faces or, with q, from the rays in q turned through the current globe (WarpDevice::warp_rays).  Every refusal
// launches nothing.
int warp_view(blinky_ctx *ctx, blinky::WarpRequest r, blinky::WarpEntry entry, int rowbytes, int x0, int y0, int keep_unmapped,
              const blinky::RayRequest *q = nullptr) {
    NEED_DEVICE(ctx);
    r.entry = entry;
    r.rowbytes = rowbytes;
    r.x0 = x0;
    r.y0 = y0;
    r.keep_unmapped = keep_unmapped != 0;
    r.rgba = entry != blinky::WarpEntry::View && entry != blinky::WarpEntry::Rays;
    const bool ok = q ? ctx->dev->warp_rays(r, *q, globe_state(ctx), ctx->host.device_params(ctx->dev->width(), ctx->dev->height(), ctx->dev->platesize()))
                      : ctx->dev->warp(r);
    return ok ? BLINKY_OK : set_err(ctx, ctx->dev->last_error_code(), ctx->dev->last_error());
}

}  // namespace

extern "C" {

int blinky_warp_device(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out, size_t out_stride,
                       int nframes, void *stream) {
    NEED_DEVICE(ctx);
    blinky::WarpRequest r(d_faces, face_stride, d_out, out_stride, nframes, stream);
    r.entry = blinky::WarpEntry::Dense;
    return ctx->dev->warp(r) ? BLINKY_OK : set_err(ctx, ctx->dev->last_error_code(), ctx->dev->last_error());
}

int blinky_warp_device_view(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_screen, size_t screen_frame_stride,
                            int rowbytes, int x0, int y0, int nframes, int keep_unmapped, void *stream) {
    return warp_view(ctx, {d_faces, face_stride, d_screen, screen_frame_stride, nframes, stream}, blinky::WarpEntry::View, rowbytes, x0, y0,
                     keep_unmapped);
}

int blinky_warp_device_view_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_screen, size_t screen_frame_stride,
                                 int rowbytes, int x0, int y0, int nframes, int keep_unmapped, void *stream) {
    return warp_view(ctx, {d_faces, face_stride, d_screen, screen_frame_stride, nframes, stream}, blinky::WarpEntry::ViewRgba, rowbytes, x0,
                     y0, keep_unmapped);
}

int blinky_warp_device_view_rgba_tables(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_screen_rgba,
                                        size_t screen_frame_stride, int rowbytes, int x0, int y0, int nframes, int keep_unmapped,
                                        const uint32_t *d_tables, size_t table_stride, void *stream) {
    blinky::WarpRequest r(d_faces, face_stride, d_screen_rgba, screen_frame_stride, nframes, stream);
    r.tables = d_tables;
    r.table_stride = table_stride;
    return warp_view(ctx, r, blinky::WarpEntry::ViewRgbaTables, rowbytes, x0, y0, keep_unmapped);
}

int blinky_warp_device_rays(blinky_ctx *ctx, const void *d_faces, size_t face_stride, const float *d_rays, size_t ray_stride, const float *d_xforms,
                            size_t xform_stride, void *d_screen, size_t screen_frame_stride, int rowbytes, int x0, int y0, int nframes,
                            int keep_unmapped, void *stream) {
    const blinky::RayRequest q = {d_rays, ray_stride, d_xforms, xform_stride};
    return warp_view(ctx, {d_faces, face_stride, d_screen, screen_frame_stride, nframes, stream}, blinky::WarpEntry::Rays, rowbytes, x0, y0,
                     keep_unmapped, &q);
}

int blinky_warp_device_rays_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, const float *d_rays, size_t ray_stride,
                                 const float *d_xforms, size_t xform_stride, void *d_screen_rgba, size_t screen_frame_stride, int rowbytes,
                                 int x0, int y0, int nframes, int keep_unmapped, const uint32_t *d_tables, size_t table_stride, void *stream) {
    blinky::WarpRequest r(d_faces, face_stride, d_screen_rgba, screen_frame_stride, nframes, stream);
    r.tables = d_tables;
    r.table_stride = table_stride;
    const blinky::RayRequest q = {d_rays, ray_stride, d_xforms, xform_stride};
    return warp_view(ctx, r, blinky::WarpEntry::RaysRgba, rowbytes, x0, y0, keep_unmapped, &q);
}

int blinky_warp_device_rays_supersampled(blinky_ctx *ctx, const void *d_faces, size_t face_stride, const float *d_rays, size_t ray_stride,
                                         const float *d_xforms, size_t xform_stride, int factor, void *d_screen_rgba, size_t screen_frame_stride,
                                         int rowbytes, int x0, int y0, int nframes, int keep_unmapped, const uint32_t *d_tables, size_t table_stride,
                                         void *stream) {
    blinky::WarpRequest r(d_faces, face_stride, d_screen_rgba, screen_frame_stride, nframes, stream);
    r.tables = d_tables;
    r.table_stride = table_stride;
    blinky::RayRequest q = {d_rays, ray_stride, d_xforms, xform_stride};
    q.factor = factor;
    return warp_view(ctx, r, blinky::WarpEntry::RaysSupersampled, rowbytes, x0, y0, keep_unmapped, &q);
}

int blinky_warp_device_rays_bilinear(blinky_ctx *ctx, const void *d_faces, size_t face_stride, const float *d_rays, size_t ray_stride,
                                     const float *d_xforms, size_t xform_stride, int factor, void *d_screen_rgba, size_t screen_frame_stride,
                                     int rowbytes, int x0, int y0, int nframes, int keep_unmapped, const uint32_t *d_tables, size_t table_stride,
                                     void *stream) {
    blinky::WarpRequest r(d_faces, face_stride, d_screen_rgba, screen_frame_stride, nframes, stream);
    r.tables = d_tables;
    r.table_stride = table_stride;
    blinky::RayRequest q = {d_rays, ray_stride, d_xforms, xform_stride};
    q.factor = factor;
    q.filter = blinky::RayFilter::Bilinear;
    return warp_view(ctx, r, blinky::WarpEntry::RaysBilinear, rowbytes, x0, y0, keep_unmapped, &q);
}

int blinky_ray_pyramid_bytes(blinky_ctx *ctx, size_t *bytes) {
    NEED_DEVICE(ctx);
    const char *who = "blinky_ray_pyramid_bytes";
    if (!bytes) return set_err(ctx, BLINKY_E_INVALID, std::string(who) + ": NULL bytes");
    blinky::WarpRequest r(nullptr, 0, nullptr, 0, 0, nullptr);
    r.entry = blinky::WarpEntry::PyramidBytes;
    blinky::CheckedWarp c;
    const int rc = blinky::check_warp(r, blinky::RayRequest(), ctx->dev->state(globe_state(ctx)), &c, &ctx->err);
    if (rc == BLINKY_OK) *bytes = static_cast<size_t>(c.pyramid_bytes);
    return rc;
}

int blinky_warp_device_rays_trilinear(blinky_ctx *ctx, const void *d_faces, size_t face_stride, const float *d_rays, size_t ray_stride,
                                      const float *d_xforms, size_t xform_stride, void *d_screen_rgba, size_t screen_frame_stride, int rowbytes,
                                      int x0, int y0, int nframes, int keep_unmapped, const uint32_t *d_tables, size_t table_stride,
                                      void *d_scratch, size_t scratch_bytes, void *stream) {
    blinky::WarpRequest r(d_faces, face_stride, d_screen_rgba, screen_frame_stride, nframes, stream);
    r.tables = d_tables;
    r.table_stride = table_stride;
    blinky::RayRequest q = {d_rays, ray_stride, d_xforms, xform_stride};
    q.filter = blinky::RayFilter::Trilinear;
    q.scratch = d_scratch;
    q.scratch_bytes = scratch_bytes;
    return warp_view(ctx, r, blinky::WarpEntry::RaysTrilinear, rowbytes, x0, y0, keep_unmapped, &q);
}

int blinky_warp_host(blinky_ctx *ctx, const uint8_t *faces_host, size_t face_stride, uint8_t *dst_host,
                     size_t dst_frame_stride, int dst_rowbytes, int x0, int y0, int nframes, int keep_unmapped) {
    NEED_DEVICE(ctx);
    blinky::WarpRequest r(faces_host, face_stride, dst_host, dst_frame_stride, nframes, nullptr);
    r.entry = blinky::WarpEntry::Host;
    r.rowbytes = dst_rowbytes;
    r.x0 = x0;
    r.y0 = y0;
    r.keep_unmapped = keep_unmapped != 0;
    return ctx->dev->warp_host(r) ? BLINKY_OK : set_err(ctx, ctx->dev->last_error_code(), ctx->dev->last_error());
}

int64_t blinky_upload_bytes_per_frame(blinky_ctx *ctx) {
    int64_t n = 0;
    if (!ctx->host.built()) return 0;
    for (int i = 0; i < ctx->host.map_numplates(); ++i) {
        const int *r = ctx->host.plate_rect(i);
        if (ctx->host.plate(i).display && r[0] <= r[2] && r[1] <= r[3]) n += static_cast<int64_t>(r[2] - r[0] + 1) * (r[3] - r[1] + 1);
    }
    return n;
}

int blinky_alloc_pinned(blinky_ctx *ctx, size_t bytes, void **out) {
    NEED_DEVICE(ctx);
    return ctx->dev->alloc_pinned(bytes, out) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_free_pinned(blinky_ctx *ctx, void *ptr) {
    NEED_DEVICE(ctx);
    return ctx->dev->free_pinned(ptr) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_alloc_device(blinky_ctx *ctx, size_t bytes, void **out) {
    NEED_DEVICE(ctx);
    return ctx->dev->alloc_device(bytes, out) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_free_device(blinky_ctx *ctx, void *ptr) {
    NEED_DEVICE(ctx);
    return ctx->dev->free_device(ptr) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_ipc_export(blinky_ctx *ctx, void *device_ptr, unsigned char handle[64]) {
    NEED_DEVICE(ctx);
    return ctx->dev->ipc_export(device_ptr, handle) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_ipc_open(blinky_ctx *ctx, const unsigned char handle[64], void **peer_ptr) {
    NEED_DEVICE(ctx);
    return ctx->dev->ipc_open(handle, peer_ptr) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_ipc_close(blinky_ctx *ctx, void *peer_ptr) {
    NEED_DEVICE(ctx);
    return ctx->dev->ipc_close(peer_ptr) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_sync(blinky_ctx *ctx) {
    NEED_DEVICE(ctx);
    return ctx->dev->sync() ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}
int blinky_release_captures(blinky_ctx *ctx) {
    NEED_DEVICE(ctx);
    return ctx->dev->release_captures() ? BLINKY_OK : set_err(ctx, ctx->dev->last_error_code(), ctx->dev->last_error());
}

int blinky_set_rgba_table(blinky_ctx *ctx, const uint32_t table[256]) {
    NEED_DEVICE(ctx);
    return ctx->dev->set_rgba_table(table) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

int blinky_warp_device_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out, size_t out_stride,
                            int nframes, void *stream) {
    NEED_DEVICE(ctx);
    blinky::WarpRequest r(d_faces, face_stride, d_out, out_stride, nframes, stream);
    r.entry = blinky::WarpEntry::DenseRgba;
    r.rgba = true;
    return ctx->dev->warp(r) ? BLINKY_OK : set_err(ctx, ctx->dev->last_error_code(), ctx->dev->last_error());
}

int64_t blinky_launch_count(blinky_ctx *ctx) { return ctx->dev ? ctx->dev->launches() : 0; }
const char *blinky_plan_summary(blinky_ctx *ctx) {
    if (!ctx->host.built() || !host_map(ctx)) return "";
    blinky::TilePlan pl = current_plan(ctx, 1);
    const double npix = static_cast<double>(ctx->host.width()) * ctx->host.height();
    char buf[256];
    snprintf(buf, sizeof buf, "tiles %dx%d of %dx%d px: %d box (%d fully mapped; TMA, %.3f B/px staged, %zu shapes), %d gather, %d empty; entries %.3f B/px",
             pl.tiles_x, pl.tiles_y, blinky::kTileW, blinky::kTileH, pl.n_box, pl.n_box_full, static_cast<double>(pl.box_bytes) / npix,
             pl.shapes.size(), pl.n_gather, pl.n_empty, static_cast<double>(pl.entries.size()) / npix);
    ctx->scratch = buf;
    return ctx->scratch.c_str();
}
int blinky_get_tile_plan(blinky_ctx *ctx, void *tiles_out, size_t tiles_cap, void *entries_out, size_t entries_cap, size_t *ntiles,
                         size_t *entry_bytes) {
    if (!ctx->host.built()) return set_err(ctx, BLINKY_E_STATE, "no lensmap built");
    if (ctx->device_plan) {
        // the plan the GPU planner wrote, as the kernels read it
        const size_t nt = ctx->dev->plan_tiles(), nb = ctx->dev->plan_entry_bytes();
        if (ntiles) *ntiles = nt;
        if (entry_bytes) *entry_bytes = nb;
        if (tiles_out && tiles_cap < nt * sizeof(blinky::TileDesc)) return set_err(ctx, BLINKY_E_INVALID, "tile buffer too small");
        if (entries_out && entries_cap < nb) return set_err(ctx, BLINKY_E_INVALID, "entry buffer too small");
        return ctx->dev->download_plan(tiles_out, entries_out, entries_out ? nb : 0) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
    }
    if (!host_map(ctx)) return BLINKY_E_CUDA;
    blinky::TilePlan pl = current_plan(ctx, ctx->host.worker_threads());
    if (ntiles) *ntiles = pl.tiles.size();
    if (entry_bytes) *entry_bytes = pl.entries.size();
    if (tiles_out) {
        if (tiles_cap < pl.tiles.size() * sizeof(blinky::TileDesc)) return set_err(ctx, BLINKY_E_INVALID, "tile buffer too small");
        memcpy(tiles_out, pl.tiles.data(), pl.tiles.size() * sizeof(blinky::TileDesc));
    }
    if (entries_out) {
        if (entries_cap < pl.entries.size()) return set_err(ctx, BLINKY_E_INVALID, "entry buffer too small");
        memcpy(entries_out, pl.entries.data(), pl.entries.size());
    }
    return BLINKY_OK;
}

uint64_t blinky_plan_digest(blinky_ctx *ctx, int threads) {
    if (!ctx->host.built() || !host_map(ctx)) return 0;
    blinky::TilePlan pl = current_plan(ctx, threads);
    uint64_t h = 1469598103934665603ull;  // FNV-1a over the tile table and the entry blocks
    auto mix = [&](const void *p, size_t n) {
        const unsigned char *b = static_cast<const unsigned char *>(p);
        for (size_t i = 0; i < n; ++i) h = (h ^ b[i]) * 1099511628211ull;
    };
    mix(pl.tiles.data(), pl.tiles.size() * sizeof(blinky::TileDesc));
    mix(pl.entries.data(), pl.entries.size());
    return h;
}
const char *blinky_last_kernel(blinky_ctx *ctx) { return ctx->dev ? ctx->dev->last_kernel().c_str() : ""; }

// ---- sharded batches ---------------------------------------------------------------------
int blinky_shard_range(int total_frames, int rank, int world, int *first, int *count) {
    if (world < 1 || rank < 0 || rank >= world || total_frames < 0) return BLINKY_E_INVALID;
    blinky::shard_range(total_frames, rank, world, first, count);
    return BLINKY_OK;
}

int blinky_shard_unique_id(unsigned char id[128]) {
    std::string err;
    if (!id) return BLINKY_E_INVALID;
    if (!blinky::ShardGroup::unique_id(id, err)) {
        fprintf(stderr, "blinky_shard_unique_id: %s\n", err.c_str());
        return BLINKY_E_CUDA;
    }
    return BLINKY_OK;
}

int blinky_shard_init(blinky_ctx *ctx, int rank, int world, const unsigned char id[128]) {
    NEED_DEVICE(ctx);
    if (!id) return set_err(ctx, BLINKY_E_INVALID, "blinky_shard_init: id is NULL");
    if (ctx->shard) return set_err(ctx, BLINKY_E_STATE, "blinky_shard_init: already initialised (blinky_shard_close first)");
    std::unique_ptr<blinky::ShardGroup> g(new blinky::ShardGroup(ctx->dev.get(), ctx->dev->device()));
    if (!g->init(rank, world, id)) return set_err(ctx, BLINKY_E_CUDA, g->last_error());
    ctx->shard = std::move(g);
    return BLINKY_OK;
}

int blinky_shard_buffer(blinky_ctx *ctx, int total_frames, void **root_buffer) {
    NEED_DEVICE(ctx);
    if (!ctx->shard) return set_err(ctx, BLINKY_E_STATE, "blinky_shard_buffer: call blinky_shard_init first");
    if (!ctx->host.built()) return set_err(ctx, BLINKY_E_STATE, "blinky_shard_buffer: build a lensmap first (the frames have the view's size)");
    if (total_frames < 0) return set_err(ctx, BLINKY_E_INVALID, "blinky_shard_buffer: total_frames < 0");
    const size_t fb = static_cast<size_t>(ctx->host.width()) * ctx->host.height();
    return ctx->shard->buffer(total_frames, fb, root_buffer) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->shard->last_error());
}

int blinky_shard_warp_gather(blinky_ctx *ctx, const void *d_faces, size_t face_stride, int total_frames, int mode, int chunk_frames,
                             void *stream) {
    NEED_DEVICE(ctx);
    if (!ctx->shard) return set_err(ctx, BLINKY_E_STATE, "blinky_shard_warp_gather: call blinky_shard_init first");
    return ctx->shard->warp_gather(d_faces, face_stride, total_frames, mode, chunk_frames, stream)
               ? BLINKY_OK
               : set_err(ctx, BLINKY_E_CUDA, ctx->shard->last_error());
}

int blinky_shard_sync(blinky_ctx *ctx) {
    NEED_DEVICE(ctx);
    if (!ctx->shard) return set_err(ctx, BLINKY_E_STATE, "blinky_shard_sync: no shard group");
    return ctx->shard->sync() ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->shard->last_error());
}

int blinky_shard_close(blinky_ctx *ctx) {
    ctx->shard.reset();
    return BLINKY_OK;
}

}  // extern "C"
