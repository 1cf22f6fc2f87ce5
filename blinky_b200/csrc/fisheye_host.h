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
    void set_device_builder(LensDevice *b) { device_builder_ = b; }
    // host threads for the fallback evaluation and for the per-pixel passes after the map is known
    void set_worker_threads(int n) { fallback_threads_ = n < 1 ? 1 : n; }
    int worker_threads() const { return fallback_threads_; }
    // one line about how the last lensmap was built ("device: ..." / "host: ...")
    const std::string &build_info() const { return build_info_; }
    bool needs_rebuild(int width, int height, int platesize) const;

    // ---- supplied lensmaps -------------------------------------------------------
    // A caller's map replaces the current one as a build would (the lens, globe, zoom and rubix settings stay;
    // the lens / globe / zoom change flags are consumed).  Entries without BLINKY_LM_VALID are stored unmapped
    // whatever their other bits hold.  False, changing nothing, with the reason in *why, for a bad size, a NULL
    // map, an index outside the plates or a tint of 6.
    bool set_lensmap(int width, int height, int platesize, int numplates, const uint32_t *packed, std::string *why);
    // the checks of set_lensmap that do not read the map
    static bool check_lensmap_size(int width, int height, int platesize, int numplates, std::string *why);
    // What a device planner derived from a map it checked and normalised itself (tile_plan_device.h): the state
    // set_lensmap would compute, without the map.  The map follows with fill_lensmap when a query needs it.
    void adopt_lensmap(int width, int height, int platesize, int numplates, const int display[kMaxPlates], const int rect[kMaxPlates][4],
                       int64_t mapped, std::vector<int32_t> span_off, std::vector<int32_t> spans);
    bool map_on_host() const { return map_on_host_; }
    void fill_lensmap(std::vector<uint32_t> normalised);  // [height][width] entries as adopt_lensmap's planner stored them
    // plates of the current lensmap: the globe's at a build, the caller's for a supplied map
    int map_numplates() const { return map_plates_; }

    // ---- ray maps ------------------------------------------------------------------
    // A field of view rays in place of the lens: width * height float32 triples, row-major, each lens_inverse's result
    // narrowed to float and NOT normalised (normalize3 is applied here, as the build applies it; the zero vector is a
    // pixel the lens leaves empty).  The rays go through the current globe (plate choice or globe_plate, stale plate
    // slots, rubix grid) exactly as a build's rays do.  The lens, zoom and scale stay; the lens / globe / zoom change
    // flags are consumed.  check_raymap: 0, or -1 for a bad size / -7 without a valid globe (reason in *why);
    // platesize <= 0 becomes min(width, height).
    int check_raymap(int width, int height, int *platesize, std::string *why) const;
    // the host path on the worker threads: 0 ok; -2, changing nothing, when globe_plate raises an error
    int set_raymap(int width, int height, int platesize, const float *rays);
    // The device path (sizes checked): the map of the rays at d_rays (device memory, read on `stream`) in the device
    // builder's map (*d_map), with the pixels the device could not decide settled here (*settled).  0 ok; 1 = not
    // possible on the device (why): take the host path; -2 = globe_plate raised an error.  Changes no host state.
    int raymap_device(int width, int height, int platesize, const float *d_rays, void *stream, uint32_t **d_map, size_t *settled,
                      std::string *why);
    // C++ / CUDA source the ray-map kernel is appended to: the globe's globe_plate translated alone, or the bare
    // prelude for globes without one; false + reason when globe_plate does not translate
    bool raymap_device_source(bool cuda, std::string *source, std::string *why);

    // ---- ray export ------------------------------------------------------------------
    // The view rays a width x height build evaluates, as set_raymap reads them: pixel (lx, ly) gets
    // lens_inverse((lx - width/2) * scale, -(ly - height/2) * scale) (integer /2) narrowed to float and not normalised,
    // (0, 0, 0) for nil, at rays[3 * (ly * width + lx)].  The loaded lens_inverse is evaluated (the script is not re-run)
    // and no globe is needed.  Nothing of the context changes: not the map, the scale or the change flags.
    // check_rays: 0 with the scale calc_zoom gives for width x height in *scale; -7 without a valid lens that has a
    // per-pixel ray (reason in *why); -3 when the zoom fails (the build's console message is printed).
    int check_rays(int width, int height, double *scale, std::string *why);
    // the host path on the worker threads: 0 ok; -2 when lens_inverse raises an error or returns a bad result
    int export_rays(int width, int height, double scale, float *rays);
    // The device path: the rays into d_rays (device memory) on `stream`, the pixels the device could not decide evaluated
    // here (*settled).  0 ok, the field complete; 1 = not possible on the device (why): take the host path; -2 as
    // export_rays.
    int export_rays_device(int width, int height, double scale, float *d_rays, void *stream, size_t *settled, std::string *why);

    // ---- ray export of a forward lens (DESIGN §3h) ------------------------------------------------------------------
    // The view rays of a width x height forward build on plates of platesize texels, at the scale calc_zoom gives:
    // each pixel the build maps gets the ray through the point of its winning texel's quad where the pixel lies
    // (forward_raster.h: fwd_quad_ray), normalised; the others get (0, 0, 0).  Same layout as export_rays.  The build's
    // grid points, stale slots, texel owners and maxdiff guard apply; nothing is printed and nothing of the context
    // changes.  check_rays_forward: platesize <= 0 becomes min(width, height); 0 with the scale in *scale; -1 for a
    // platesize beyond the 28-bit texel index; -7 without a valid lens, a lens_forward function or a valid globe
    // (reason in *why); -3 when the zoom fails (the build's console message is printed).
    int check_rays_forward(int width, int height, int *platesize, double *scale, std::string *why);
    // the host path: the serial forward builder; 0 ok, -2 when lens_forward or globe_plate fails
    int export_rays_forward(int width, int height, int platesize, double scale, float *rays);
    // the device path: the rays into d_rays (device memory) on `stream`, with *settled grid points and texel owners
    // settled by the interpreter.  0 ok; 1 = not possible on the device (why): take the host path; -2 as the host path.
    int export_rays_forward_device(int width, int height, int platesize, double scale, float *d_rays, void *stream, size_t *settled,
                                   std::string *why);

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
    // the globe picks its plates with a globe_plate script (whose decisions can need the interpreter)
    bool has_globe_plate() const { return fn_globe_plate_.is_function(); }
    // the globe's plates, rubix grid and uv scales (and the lens's scale) as the device kernels read them, for a
    // width x height view on plates of platesize texels
    LensBuildParams device_params(int width, int height, int platesize) const;
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
    // rowbytes > 0: the faces follow a face layout (face_layout.h) with the plates' (x, y) origins
    std::vector<uint8_t> plate_pcx(const uint8_t *faces, int plate, bool with_margins, int rowbytes = 0, const int32_t *origins = nullptr);
    // writes <dir>/<name><i>.pcx for every plate, prints "Wrote ..." and disarms the request
    bool save_globe(const uint8_t *faces, const std::string &dir, int rowbytes = 0, const int32_t *origins = nullptr);

    // raw script probes: 1 = values, 0 = nil, -1 = bad return, -2 = no such function, -3 = script error
    int lens_inverse(double x, double y, double out[3]);
    int lens_forward(double rx, double ry, double rz, double *x, double *y);
    // the globe's globe_plate(x, y, z) as ray_to_plate_index reads it: 1 = a number (*plate =
    // (int)(ptrdiff_t) of the last value returned), 0 = no value / nil / not a number (*plate = -1)
    int globe_plate(double x, double y, double z, int *plate);

    // C++/CUDA source of the current lens_inverse (lua_transpile.h); false + reason when the
    // lens is outside the transpilable subset.  with_globe_plate: a globe_plate script of the globe is
    // translated into the same unit (what the device builder compiles)
    bool lens_device_source(bool cuda, std::string *source, std::string *why, bool forward = false, bool with_globe_plate = false);
    // the globe's globe_plate translated alone; false + reason when there is none or it does not translate
    bool globe_plate_device_source(bool cuda, std::string *source, std::string *why);

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
    bool calc_zoom(int width, int height, double *scale);  // the scale of a width x height build; false + console message
    void create_palmap();
    int find_closest_pal_index(int r, int g, int b) const;

    int ray_to_plate_index(Worker &w, const float ray[3]);
    bool ray_to_plate_uv(int plate, const float ray[3], double *u, double *v) const;
    bool on_rubix_grid(int px, int py, int ps) const;
    void set_from_plate(int lx, int ly, int px, int py, int plate, int *display);
    bool ray_to_texel(Worker &w, const float ray[3], int ps, int *plate, int *px, int *py);
    void set_from_ray(Worker &w, int lx, int ly, const float ray[3], int *display);
    uint32_t ray_entry(Worker &w, const float ray[3], int ps, int *display);
    int call_inverse(Worker &w, double x, double y, float ray[3]);
    int eval_inverse(Worker &w, double x, double y, float ray[3]);
    int call_forward(Worker &w, const float ray[3], double *x, double *y);
    int build_inverse_rows(Worker &w, int y_begin, int y_end, int *display);  // rows [y_begin,y_end), bottom-up
    int build_inverse_pixels(Worker &w, const int32_t *pixels, size_t n, int *display);
    // runs item(w, i, display) for i in [0, nitems) over `threads` cloned script states
    template <class F>
    int run_inverse_workers(int threads, int nitems, int *display, F item);
    // the interpreter's share of a device build: chunk(w, b, e, display) for the items [b, e) of n the device left to
    // the host, 256 at a time, on one thread below 4096 items and on the fallback threads from there
    template <class F>
    int settle_flagged(size_t n, int *display, F chunk);
    int build_inverse(int threads);
    int build_inverse_device(int *display, std::string *why);  // 0 ok, -1 script failure, 1 = not possible (why)
    int build_forward_device(std::string *why);                // same convention
    int build_forward(int threads);
    struct ForwardView {  // the geometry of a forward build
        int width, height, ps;
        double scale;
    };
    int forward_device_points(const ForwardView &fv, std::vector<ForwardPatch> *patches, std::vector<uint32_t> *owner_patches, std::string *why);
    template <class Sink>
    int forward_loop(const ForwardView &fv, Sink &sink);
    int uv_to_screen(Worker &w, const ForwardView &fv, int plate, double u, double v, int *lx, int *ly);
    template <class Sink>
    void draw_quad(const int *tl, const int *tr, const int *bl, const int *br, Sink &sink);
    void finish_build();
    void unpack_map(const uint32_t *packed);

    // Lua-visible C functions
    static void lua_latlon_to_ray(minilua::State &, const minilua::Value *, int, minilua::ValueList &, void *);
    static void lua_ray_to_latlon(minilua::State &, const minilua::Value *, int, minilua::ValueList &, void *);
    static void lua_plate_to_ray(minilua::State &, const minilua::Value *, int, minilua::ValueList &, void *);
    static void lua_print_sink(const char *text, void *ud);

    std::unique_ptr<minilua::State> lua_;
    minilua::Value fn_inverse_, fn_forward_, fn_globe_plate_;  // registry refs, :328-332

    LensDevice *device_builder_ = nullptr;  // not owned
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
    bool map_on_host_ = true;  // false after adopt_lensmap until fill_lensmap: idx_ / tint_ / packed_ are not the map yet
    int map_plates_ = 0;
    int built_w_ = -1, built_h_ = -1, built_ps_ = -1;
    std::vector<int32_t> idx_;
    std::vector<uint8_t> tint_;
    std::vector<uint32_t> packed_;
    std::vector<int32_t> span_off_, spans_;
    int64_t mapped_ = 0;
    int plate_rect_[kMaxPlates][4];
};

}  // namespace blinky
