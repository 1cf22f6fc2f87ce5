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
#include "lens_device.h"
#include "shard.h"
#include "tile_plan.h"
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
    uint8_t palmaps[BLINKY_MAX_PLATES * 256];
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

bool upload(blinky_ctx *c) {
    if (!c->dev || !c->host.built()) return true;
    blinky::LensmapUpload lm;
    lm.width = c->host.width();
    lm.height = c->host.height();
    lm.platesize = c->host.platesize();
    lm.numplates = c->host.numplates();
    lm.packed = c->host.packed().data();
    for (int i = 0; i < BLINKY_MAX_PLATES; ++i) {
        memcpy(c->palmaps + i * 256, c->host.plate(i).palette, 256);
        lm.display[i] = i < c->host.numplates() ? c->host.plate(i).display : 0;
        memcpy(lm.plate_rect[i], c->host.plate_rect(i), sizeof lm.plate_rect[i]);
    }
    lm.palmaps = c->palmaps;
    lm.rubix = c->host.rubix_enabled();
    lm.span_off = c->host.row_span_offsets().data();
    lm.spans = c->host.row_spans().data();
    lm.nspans = c->host.row_spans().size() / 2;
    // TMA needs 16-byte aligned plate rows; other plate sizes use direct gathers only
    blinky::TilePlan plan = blinky::make_tile_plan(lm.packed, lm.width, lm.height, lm.platesize, lm.platesize % 16 == 0, c->host.worker_threads());
    lm.plan = &plan;
    if (!c->dev->upload_lensmap(lm)) {
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
    memset(c->palmaps, 0, sizeof c->palmaps);
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
    if (!upload(ctx)) return BLINKY_E_CUDA;
    return BLINKY_OK;
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

const char *blinky_build_info(blinky_ctx *ctx) { return ctx->build_info.c_str(); }

int blinky_compile_lens(blinky_ctx *ctx, int forward, size_t *cubin_bytes) {
    std::string src, why;
    if (!ctx->host.lens_device_source(true, &src, &why, forward != 0)) return set_err(ctx, BLINKY_E_SCRIPT, why);
    std::vector<char> cubin;
    std::string log;
    if (!LensDevice::compile(src, forward != 0, &cubin, &log)) return set_err(ctx, BLINKY_E_CUDA, log);
    if (cubin_bytes) *cubin_bytes = cubin.size();
    return BLINKY_OK;
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
    for (int i = 0; i < BLINKY_MAX_PLATES; ++i) out[i] = i < ctx->host.numplates() ? ctx->host.plate(i).display : 0;
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
    if (idx) memcpy(idx, ctx->host.indices().data(), ctx->host.indices().size() * sizeof(int32_t));
    if (tint) memcpy(tint, ctx->host.tints().data(), ctx->host.tints().size());
    return BLINKY_OK;
}

int blinky_get_lensmap_packed(blinky_ctx *ctx, uint32_t *out) {
    if (!ctx->host.built()) return set_err(ctx, BLINKY_E_STATE, "no lensmap built");
    memcpy(out, ctx->host.packed().data(), ctx->host.packed().size() * sizeof(uint32_t));
    return BLINKY_OK;
}

int64_t blinky_mapped_pixels(blinky_ctx *ctx) { return ctx->host.mapped_pixels(); }

int blinky_lens_inverse(blinky_ctx *ctx, double x, double y, double ray_out[3]) { return ctx->host.lens_inverse(x, y, ray_out); }
int blinky_lens_forward(blinky_ctx *ctx, double rx, double ry, double rz, double *x, double *y) {
    return ctx->host.lens_forward(rx, ry, rz, x, y);
}

int blinky_lens_source(blinky_ctx *ctx, int flavour, char *buf, size_t bufsize) {
    std::string s, why;
    if (!ctx->host.lens_device_source((flavour & 1) != 0, &s, &why, (flavour & 2) != 0)) return set_err(ctx, BLINKY_E_SCRIPT, why);
    if (flavour & 4) s += LensDevice::kernel_tail((flavour & 2) != 0);
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

int blinky_saveglobe_pending(blinky_ctx *ctx) { return ctx->host.saveglobe_pending() ? 1 : 0; }
int blinky_save_globe(blinky_ctx *ctx, const uint8_t *faces_host, const char *directory) {
    if (!faces_host) return set_err(ctx, BLINKY_E_INVALID, "faces is NULL");
    if (!ctx->host.built()) return set_err(ctx, BLINKY_E_STATE, "no lensmap built (plate size unknown)");
    return ctx->host.save_globe(faces_host, directory ? directory : "") ? BLINKY_OK
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

int blinky_set_background(blinky_ctx *ctx, const uint8_t *bg) {
    NEED_DEVICE(ctx);
    return ctx->dev->set_background(bg) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

int blinky_warp_device(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out, size_t out_stride,
                       int nframes, void *stream) {
    NEED_DEVICE(ctx);
    return ctx->dev->warp(d_faces, face_stride, d_out, out_stride, nframes, stream, false)
               ? BLINKY_OK
               : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

int blinky_warp_host(blinky_ctx *ctx, const uint8_t *faces_host, size_t face_stride, uint8_t *dst_host,
                     size_t dst_frame_stride, int dst_rowbytes, int x0, int y0, int nframes, int keep_unmapped) {
    NEED_DEVICE(ctx);
    if (!faces_host || !dst_host) return set_err(ctx, BLINKY_E_INVALID, "NULL buffer");
    if (dst_rowbytes < ctx->host.width() + x0) return set_err(ctx, BLINKY_E_INVALID, "dst_rowbytes too small for the view rectangle");
    return ctx->dev->warp_host(faces_host, face_stride, dst_host, dst_frame_stride, dst_rowbytes, x0, y0, nframes, keep_unmapped != 0)
               ? BLINKY_OK
               : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

int64_t blinky_upload_bytes_per_frame(blinky_ctx *ctx) {
    int64_t n = 0;
    if (!ctx->host.built()) return 0;
    for (int i = 0; i < ctx->host.numplates(); ++i) {
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

int blinky_set_rgba_table(blinky_ctx *ctx, const uint32_t table[256]) {
    NEED_DEVICE(ctx);
    return ctx->dev->set_rgba_table(table) ? BLINKY_OK : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

int blinky_warp_device_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out, size_t out_stride,
                            int nframes, void *stream) {
    NEED_DEVICE(ctx);
    return ctx->dev->warp(d_faces, face_stride, d_out, out_stride, nframes, stream, true)
               ? BLINKY_OK
               : set_err(ctx, BLINKY_E_CUDA, ctx->dev->last_error());
}

int64_t blinky_launch_count(blinky_ctx *ctx) { return ctx->dev ? ctx->dev->launches() : 0; }
const char *blinky_plan_summary(blinky_ctx *ctx) {
    if (!ctx->host.built()) return "";
    blinky::TilePlan pl = blinky::make_tile_plan(ctx->host.packed().data(), ctx->host.width(), ctx->host.height(),
                                                 ctx->host.platesize(), ctx->host.platesize() % 16 == 0);
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
    blinky::TilePlan pl = blinky::make_tile_plan(ctx->host.packed().data(), ctx->host.width(), ctx->host.height(),
                                                 ctx->host.platesize(), ctx->host.platesize() % 16 == 0, ctx->host.worker_threads());
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
    if (!ctx->host.built()) return 0;
    blinky::TilePlan pl = blinky::make_tile_plan(ctx->host.packed().data(), ctx->host.width(), ctx->host.height(),
                                                 ctx->host.platesize(), ctx->host.platesize() % 16 == 0, threads);
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
