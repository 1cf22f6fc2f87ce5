// Host side of the H100 lens-warp path: everything the reference's
// engine/NQ/fisheye.c does BEFORE the per-frame gather — the Lua script
// environment, globe/lens loading, the console command surface, zoom, the rubix
// palette and the one-shot lensmap build — with the lensmap produced both in the
// reference's terms (texel index / tint byte per pixel) and in the packed 32-bit
// form the CUDA kernels read.  No CUDA in this file: it is usable (and tested)
// on a machine without a GPU.
//
// Reference map (all the reference's engine/NQ/fisheye.c): state structs
// :306-528, F_Init :642-676, console commands :916-1176, converters :1184-1214,
// init_lua :1222-1265, zoom :1273-1386, Lua bridge :1494-1651, loaders
// :1659-1913, setters :1922-2013, getters :2023-2066, builders :2084-2397.
#pragma once

#include <cstdarg>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "lens_device.h"
#include "minilua/minilua.h"

namespace blinky {

constexpr int kMaxPlates = 6;  // MAX_PLATES, fisheye.c:352

enum ZoomType { ZOOM_NONE = 0, ZOOM_FOV, ZOOM_VFOV, ZOOM_COVER, ZOOM_CONTAIN };  // :457
enum MapType { MAP_NONE = 0, MAP_INVERSE, MAP_FORWARD };                          // :391

struct Plate {  // one entry of globe.plates[], :353-361
    float forward[3];
    float right[3];
    float up[3];
    float fov;   // radians
    float dist;  // 0.5 / tan(fov/2)
    uint8_t palette[256];
    int display;
};

using PrintFn = void (*)(const char *text, void *user);
using ExecFn = void (*)(const char *command, void *user);

class FisheyeHost {
public:
    FisheyeHost();
    ~FisheyeHost();

    // ---- message / command plumbing ------------------------------------
    void set_print(PrintFn fn, void *user) { print_fn_ = fn; print_user_ = user; }
    void set_exec(ExecFn fn, void *user) { exec_fn_ = fn; exec_user_ = user; }
    void print(const char *fmt, ...) __attribute__((format(printf, 2, 3)));
    const std::string &log() const { return log_; }
    void clear_log() { log_.clear(); }

    // ---- configuration ---------------------------------------------------
    void set_basedir(const std::string &dir) { basedir_ = dir; }
    void set_palette(const uint8_t palette[768]);  // host_basepal -> create_palmap
    bool command(const std::string &line);         // console surface; false = unknown command
    bool cmd_lens(const std::string &name, const std::string *source);
    bool cmd_globe(const std::string &name, const std::string *source);
    void set_zoom(int type, int fov);
    void set_rubix(bool on) { rubix_enabled_ = on; }
    void set_rubixgrid(int numcells, double cell, double pad);

    // ---- build -------------------------------------------------------------
    // returns 0 ok; -2 script problem; -3 zoom failure; -7 invalid lens/globe.
    // threads >= 1: the lens script is interpreted on that many host threads.
    // threads == 0: evaluate the lens on the GPU when a device builder is installed and the
    // lens translates (lua_transpile.h); pixels the device cannot decide exactly, and lenses
    // outside the translatable subset, go through the interpreter on `fallback_threads`.
    int build_lensmap(int width, int height, int platesize, int threads);
    void set_device_builder(DeviceLensBuilder *b) { device_builder_ = b; }
    // host threads for the fallback evaluation and for the per-pixel passes after the map is known
    void set_worker_threads(int n) { fallback_threads_ = n < 1 ? 1 : n; }
    int worker_threads() const { return fallback_threads_; }
    // one line about how the last lensmap was built ("device: ..." / "host: ...")
    const std::string &build_info() const { return build_info_; }
    bool needs_rebuild(int width, int height, int platesize) const;

    // ---- results -------------------------------------------------------------
    int width() const { return width_px_; }
    int height() const { return height_px_; }
    int platesize() const { return platesize_; }
    int numplates() const { return numplates_; }
    const Plate &plate(int i) const { return plates_[i]; }
    double scale() const { return scale_; }
    bool built() const { return built_; }
    const std::vector<int32_t> &indices() const { return idx_; }
    const std::vector<uint8_t> &tints() const { return tint_; }
    const std::vector<uint32_t> &packed() const { return packed_; }
    int64_t mapped_pixels() const { return mapped_; }
    // per plate, the texel rectangle {x0, y0, x1, y1} (inclusive) the lens reads; x0 > x1 = unused plate
    const int *plate_rect(int plate) const { return plate_rect_[plate]; }
    // per row, the [x0,x1) spans of mapped pixels (for exact "only mapped pixels
    // are written" copy-back, render_lensmap :2413)
    const std::vector<int32_t> &row_span_offsets() const { return span_off_; }
    const std::vector<int32_t> &row_spans() const { return spans_; }

    // ---- state queries ---------------------------------------------------------
    bool fisheye_enabled() const { return fisheye_enabled_; }
    bool lens_valid() const { return lens_valid_; }
    bool globe_valid() const { return globe_valid_; }
    const std::string &lens_name() const { return lens_name_; }
    const std::string &globe_name() const { return globe_name_; }
    const std::string &onload() const { return onload_; }
    int map_type() const { return map_type_; }
    int zoom_type() const { return zoom_type_; }
    int zoom_fov() const { return zoom_fov_; }
    int max_fov() const { return max_fov_; }
    int max_vfov() const { return max_vfov_; }
    double lens_width() const { return lens_width_; }
    double lens_height() const { return lens_height_; }
    bool rubix_enabled() const { return rubix_enabled_; }
    int rubix_numcells() const { return rubix_numcells_; }
    double rubix_cell() const { return rubix_cell_; }
    double rubix_pad() const { return rubix_pad_; }
    std::string write_config() const;  // F_WriteConfig :683-696

    // f_saveglobe (:1120-1136, 1396-1486): the command only arms a request; the frame
    // driver hands the plates over once they are rendered
    bool saveglobe_pending() const { return save_pending_; }
    // PCX image of one plate exactly as WritePCXplate builds it (texels another plate
    // owns are blanked to 0xFE unless with_margins)
    std::vector<uint8_t> plate_pcx(const uint8_t *faces, int plate, bool with_margins);
    // writes <dir>/<name><i>.pcx for every plate, prints "Wrote ..." and disarms the request
    bool save_globe(const uint8_t *faces, const std::string &dir);

    // raw script probes: 1 = values, 0 = nil, -1 = bad return, -2 = no such function, -3 = script error
    int lens_inverse(double x, double y, double out[3]);
    int lens_forward(double rx, double ry, double rz, double *x, double *y);

    // C++/CUDA source of the current lens_inverse (lua_transpile.h); false + reason when the
    // lens is outside the transpilable subset
    bool lens_device_source(bool cuda, std::string *source, std::string *why, bool forward = false);

    // pure converters, exposed for the Lua-visible wrappers
    static void latlon_to_ray(double lat, double lon, float ray[3]);
    static void ray_to_latlon(const float ray[3], double *lat, double *lon);
    void plate_uv_to_ray(int plate, double u, double v, float ray[3]) const;

private:
    struct Worker;  // one Lua state + resolved function handles
    bool load_lens();
    bool load_globe();
    void clear_lens_vars();
    void clear_globe_vars();
    bool run_script(const std::string &kind, const std::string &name, const std::string *source);
    bool calc_zoom();
    void create_palmap();
    int find_closest_pal_index(int r, int g, int b) const;

    int ray_to_plate_index(Worker &w, const float ray[3]);
    bool ray_to_plate_uv(int plate, const float ray[3], double *u, double *v) const;
    void set_from_plate(int lx, int ly, int px, int py, int plate, int *display);
    void set_from_ray(Worker &w, int lx, int ly, const float ray[3], int *display);
    int call_inverse(Worker &w, double x, double y, float ray[3]);
    int call_forward(Worker &w, const float ray[3], double *x, double *y);
    int build_inverse_rows(Worker &w, int y_begin, int y_end, int *display);  // rows [y_begin,y_end), bottom-up
    int build_inverse_pixels(Worker &w, const int32_t *pixels, size_t n, int *display);
    // runs item(w, i, display) for i in [0, nitems) over `threads` cloned script states
    template <class F>
    int run_inverse_workers(int threads, int nitems, int *display, F item);
    int build_inverse(int threads);
    int build_inverse_device(int *display, std::string *why);  // 0 ok, -1 script failure, 1 = not possible (why)
    int build_forward_device(std::string *why);                // same convention
    LensBuildParams device_params() const;
    int build_forward(int threads);
    int uv_to_screen(Worker &w, int plate, double u, double v, int *lx, int *ly);
    void draw_quad(const int *tl, const int *tr, const int *bl, const int *br, int plate, int px, int py, int *display);
    void finish_build();

    // Lua-visible C functions
    static void lua_latlon_to_ray(minilua::State &, const minilua::Value *, int, minilua::ValueList &, void *);
    static void lua_ray_to_latlon(minilua::State &, const minilua::Value *, int, minilua::ValueList &, void *);
    static void lua_plate_to_ray(minilua::State &, const minilua::Value *, int, minilua::ValueList &, void *);
    static void lua_print_sink(const char *text, void *ud);

    std::unique_ptr<minilua::State> lua_;
    minilua::Value fn_inverse_, fn_forward_, fn_globe_plate_;  // registry refs, :328-332

    DeviceLensBuilder *device_builder_ = nullptr;  // not owned
    int fallback_threads_ = 1;
    std::string build_info_;

    PrintFn print_fn_ = nullptr;
    void *print_user_ = nullptr;
    ExecFn exec_fn_ = nullptr;
    void *exec_user_ = nullptr;
    std::string log_;
    std::string basedir_ = ".";

    // globals the engine reads
    bool fisheye_enabled_ = false;
    bool shortcutkeys_enabled_ = false;

    // globe
    std::string globe_name_, globe_source_;
    bool globe_from_source_ = false;
    bool globe_valid_ = false, globe_changed_ = false;
    Plate plates_[kMaxPlates];
    int numplates_ = 0;
    int platesize_ = 0;

    // lens
    std::string lens_name_, lens_source_, onload_;
    bool lens_from_source_ = false;
    bool lens_valid_ = false, lens_changed_ = false;
    int map_type_ = MAP_NONE;
    double lens_width_ = 0, lens_height_ = 0, scale_ = -1;
    int width_px_ = 0, height_px_ = 0;

    // zoom
    bool zoom_changed_ = false;
    int zoom_type_ = ZOOM_NONE, zoom_fov_ = 0, max_fov_ = 0, max_vfov_ = 0;

    // rubix
    bool rubix_enabled_ = false;
    int rubix_numcells_ = 0;
    double rubix_cell_ = 0, rubix_pad_ = 0;

    bool save_pending_ = false;
    int save_with_margins_ = 0;
    std::string save_name_;
    uint8_t basepal_[768];
    bool have_palette_ = false;

    // lensmap
    bool built_ = false;
    int built_w_ = -1, built_h_ = -1, built_ps_ = -1;
    std::vector<int32_t> idx_;
    std::vector<uint8_t> tint_;
    std::vector<uint32_t> packed_;
    std::vector<int32_t> span_off_, spans_;
    int64_t mapped_ = 0;
    int plate_rect_[kMaxPlates][4];
};

}  // namespace blinky
