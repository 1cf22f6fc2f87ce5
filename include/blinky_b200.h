/* blinky_b200 — C ABI of the H100-native Blinky lens-warp path.
 *
 * This is the thin boundary a C host (TyrQuake's fisheye seams, or a headless
 * harness) calls into.  It replaces, for the lens-warp path only, what the
 * reference keeps inside one statically linked translation unit,
 * the reference's engine/NQ/fisheye.c (public surface: engine/include/fisheye.h:4-9).
 * Plain pointers and sizes only; no C++ or torch types.
 *
 * Mapping to the reference (file:line are in the reference's engine/NQ/fisheye.c):
 *
 *   blinky_create / blinky_destroy      F_Init :642-676 / F_Shutdown :678-681 (state + Lua VM)
 *   blinky_set_palette                  create_palmap :857-908 (from host_basepal)
 *   blinky_command                      the console commands registered at :651-665
 *                                       (fisheye, f_lens, f_globe, f_fov, f_vfov, f_cover,
 *                                        f_contain, f_rubix, f_rubixgrid, f_help)
 *   blinky_load_lens[_source]           cmd_lens :1061-1103 / LUA_load_lens :1659-1750
 *   blinky_load_globe[_source]          cmd_globe :1138-1161 / LUA_load_globe :1752-1875
 *   blinky_set_zoom                     cmd_fov/vfov/cover/contain :955-965, :1032-1058
 *   blinky_set_rubix / _rubixgrid       cmd_rubix :933-937 / cmd_rubixgrid :939-953
 *   blinky_build_lensmap                the rebuild branch of F_RenderView :730-743 ->
 *                                       create_lensmap :2367-2397 (inverse :2084-2124,
 *                                       forward :2126-2338), one shot instead of time-sliced
 *   blinky_warp_*                       render_lensmap :2406-2424 (THE hot loop) on the GPU
 *   blinky_write_config                 F_WriteConfig :683-696
 *   blinky_save_globe                   save_globe / WritePCXplate :1396-1486
 *
 * Conventions: every function returns BLINKY_OK (0) or a negative BLINKY_E_*
 * code; blinky_last_error() has the message.  Nothing ever calls exit() (the
 * reference does on OOM, :723-726).  A context is single-threaded: calls on
 * one context must be serialised by the caller; use one context per GPU.
 */
#ifndef BLINKY_B200_H
#define BLINKY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BLINKY_MAX_PLATES 6 /* MAX_PLATES, fisheye.c:352 */

enum {
    BLINKY_OK = 0,
    BLINKY_E_INVALID = -1,   /* bad argument / call order */
    BLINKY_E_SCRIPT = -2,    /* lens or globe script failed to load or run */
    BLINKY_E_ZOOM = -3,      /* calc_zoom failed (fisheye.c:1293-1386) */
    BLINKY_E_NODEVICE = -4,  /* context has no GPU (created with device < 0) */
    BLINKY_E_CUDA = -5,      /* CUDA runtime error */
    BLINKY_E_NOMEM = -6,
    BLINKY_E_STATE = -7      /* lens/globe invalid or lensmap not built; no capture work counter left */
};

/* zoom.type, fisheye.c:457 */
enum { BLINKY_ZOOM_NONE = 0, BLINKY_ZOOM_FOV = 1, BLINKY_ZOOM_VFOV = 2, BLINKY_ZOOM_COVER = 3, BLINKY_ZOOM_CONTAIN = 4 };
/* lens.map_type, fisheye.c:391 */
enum { BLINKY_MAP_NONE = 0, BLINKY_MAP_INVERSE = 1, BLINKY_MAP_FORWARD = 2 };

/* Packed device lensmap entry (one per screen pixel, 4 bytes):
 *   bit 31      valid (reference: lens.pixels[i] != NULL)
 *   bits 28-30  rubix tint index 0..5, or 7 = none (reference: pixel_tints[i], 255 = none)
 *   bits 0-27   texel offset into the globe: plate*ps*ps + py*ps + px (GLOBEPIXEL, :349) */
#define BLINKY_LM_VALID 0x80000000u
#define BLINKY_LM_TINT_SHIFT 28
#define BLINKY_LM_TINT_NONE 7u
#define BLINKY_LM_INDEX_MASK 0x0FFFFFFFu

/* kernel variants (blinky_set_kernel) */
enum {
    BLINKY_KERNEL_AUTO = 0,    /* pick per lensmap from the tile classification */
    BLINKY_KERNEL_GATHER = 1,  /* direct global gather, vectorised coalesced stores */
    BLINKY_KERNEL_TMA = 2      /* ring kernel: TMA-staged face tiles in shared memory where tiles are coherent (what AUTO picks) */
};

typedef struct blinky_ctx blinky_ctx;
typedef void (*blinky_print_fn)(const char *text, void *user);   /* Con_Printf sink */
typedef void (*blinky_exec_fn)(const char *command, void *user); /* Cmd_ExecuteString hook for `onload` */

/* ---- lifecycle --------------------------------------------------------- */
/* device >= 0: CUDA device ordinal.  device < 0: host-only context (lensmap
 * build, palette, console surface work; every blinky_warp_* call fails with
 * BLINKY_E_NODEVICE — there is no CPU fallback for the hot path). */
int blinky_create(int device, blinky_ctx **out);
void blinky_destroy(blinky_ctx *ctx);
const char *blinky_last_error(blinky_ctx *ctx);
const char *blinky_version(void);

/* messages the reference sends to Con_Printf; default sink keeps them in a log */
void blinky_set_print_callback(blinky_ctx *ctx, blinky_print_fn fn, void *user);
/* where a lens script's `onload` command goes (fisheye.c:1087-1095); default:
 * this library's own blinky_command */
void blinky_set_exec_callback(blinky_ctx *ctx, blinky_exec_fn fn, void *user);
const char *blinky_log(blinky_ctx *ctx);
void blinky_log_clear(blinky_ctx *ctx);

/* ---- configuration (host side) ----------------------------------------- */
/* directory that contains lua-scripts/{globes,lenses}/ (com_basedir, :1666) */
int blinky_set_basedir(blinky_ctx *ctx, const char *basedir);
/* host_basepal: 256 RGB triplets -> six rubix tint LUTs */
int blinky_set_palette(blinky_ctx *ctx, const uint8_t palette[768]);
/* executes one console command line, e.g. "f_lens panini", "f_fov 170",
 * "f_globe cube", "f_rubix", "f_rubixgrid 10 4 1", "f_cover", "fisheye 1" */
int blinky_command(blinky_ctx *ctx, const char *text);

int blinky_load_globe(blinky_ctx *ctx, const char *name);
int blinky_load_lens(blinky_ctx *ctx, const char *name);
/* same, from source text instead of <basedir>/lua-scripts/...; the text is
 * kept and re-run on every rebuild exactly like the file would be (:737) */
int blinky_load_globe_source(blinky_ctx *ctx, const char *name, const char *lua_source);
int blinky_load_lens_source(blinky_ctx *ctx, const char *name, const char *lua_source);
int blinky_set_zoom(blinky_ctx *ctx, int zoom_type, int fov_degrees);
int blinky_set_rubix(blinky_ctx *ctx, int enabled);
int blinky_set_rubixgrid(blinky_ctx *ctx, int numcells, double cell_size, double pad_size);

/* ---- lensmap build ("InitLensMap") -------------------------------------- */
/* Builds the lensmap for a width x height view and square plates of
 * `platesize` pixels (the reference forces platesize = min(w,h), :707; pass
 * platesize <= 0 for that behaviour).
 *   threads == 1  the lens script is interpreted in the reference's own order on one
 *                 script state;
 *   threads  > 1  rows are split over that many cloned script states (requires
 *                 lens_inverse to be a pure function of x,y — true for every shipped lens);
 *   threads  < 0  as above with every CPU the process may use;
 *   threads == 0  GPU build: the lens function is translated to CUDA, compiled for sm_90a
 *                 with NVRTC and evaluated by one kernel — lens_inverse for every screen
 *                 pixel, or, for forward-only lenses, lens_forward for every plate grid point
 *                 followed by the quad rasterisation in the reference's writer order.
 *                 A globe's globe_plate script is translated with the lens and picks the
 *                 plate on the device too (for forward lenses: which plate owns each texel).
 *                 Results that are not provably the host's (error bounds on every libm call)
 *                 are re-evaluated by the interpreter, so the map is the same as the host
 *                 build's.  Lenses or globe_plate scripts outside the translatable subset and
 *                 CPU-only contexts fall back to threads < 0.
 * blinky_build_info() says which way the last build went.
 * On a GPU context the packed map, tile table and tint LUTs are uploaded too. */
int blinky_build_lensmap(blinky_ctx *ctx, int width, int height, int platesize, int threads);
/* e.g. "device: 12 of 8294400 pixels re-evaluated by the interpreter; NVRTC 310 ms, kernel 1.9 ms"
 * or "host (line 22: nil values are not supported here)" */
const char *blinky_build_info(blinky_ctx *ctx);
/* Translate + NVRTC-compile the current lens_inverse (forward = 0) or lens_forward (forward = 1)
 * kernel without running it (works without a GPU). */
int blinky_compile_lens(blinky_ctx *ctx, int forward, size_t *cubin_bytes);
/* Test hook, not for applications: runs one of the translated lenses' math wrappers on the GPU, as every
 * lens unit compiles it (the same prelude text, NVRTC and options), so a test can hold the device's
 * libm and the error bound the prelude charges against the host's libm.  For i < n: v[i] and e[i] are
 * the value and the bound of op on the exact arguments a[i] (and b[i] for the two-argument ops; d_b may
 * be NULL otherwise).  For the IEEE operations e[i] is 0, except BLINKY_PROBE_MODF, which writes the
 * fractional part to v and the integral part to e.  d_a, d_b, d_v, d_e: 8-byte aligned device memory,
 * read and written on `stream` (a cudaStream_t, NULL = the default stream) after the work already there;
 * the call returns once the results are written.  n = 0 only compiles the unit (no GPU needed; also on
 * host-only contexts).  BLINKY_E_INVALID for an unknown op or a NULL / misaligned pointer, BLINKY_E_STATE
 * while `stream` is capturing a graph, BLINKY_E_NODEVICE for n > 0 on a host-only context, BLINKY_E_CUDA
 * when NVRTC is missing or the unit does not compile. */
enum {
    BLINKY_PROBE_SIN = 0, BLINKY_PROBE_COS, BLINKY_PROBE_TAN, BLINKY_PROBE_ASIN, BLINKY_PROBE_ACOS, BLINKY_PROBE_ATAN,
    BLINKY_PROBE_ATAN2,   /* atan2(a, b) */
    BLINKY_PROBE_EXP, BLINKY_PROBE_LOG, BLINKY_PROBE_LOG10,
    BLINKY_PROBE_LOGB,    /* Lua's math.log(a, b) */
    BLINKY_PROBE_SINH, BLINKY_PROBE_COSH, BLINKY_PROBE_TANH,
    BLINKY_PROBE_POW,     /* pow(a, b) */
    /* the operations the device computes exactly as the host does (IEEE) */
    BLINKY_PROBE_SQRT, BLINKY_PROBE_FMOD, BLINKY_PROBE_FLOOR, BLINKY_PROBE_CEIL, BLINKY_PROBE_TRUNC, BLINKY_PROBE_MODF,
    BLINKY_PROBE_DIV,     /* a / b */
    BLINKY_PROBE_F32,     /* (double)(float)a */
    BLINKY_PROBE_INT,     /* (double)(int)a, for a in int range */
    BLINKY_PROBE_COUNT
};
int blinky_probe_math(blinky_ctx *ctx, int op, const double *d_a, const double *d_b, double *d_v, double *d_e, size_t n, void *stream);
/* 1 if a lens/globe/zoom/rubixgrid/size change since the last build requires a rebuild (:730) */
int blinky_needs_rebuild(blinky_ctx *ctx, int width, int height, int platesize);

/* Supplied lensmaps: a map the caller made (a calibrated projector or dome warp exported by another
 * tool, a lens the host evaluates itself, a zoom or morph computed by the host's own kernel) replaces
 * the current lensmap as a build would.  map: width*height entries in the BLINKY_LM_* format,
 * row-major, dense (row pitch = width), indexing numplates plates of platesize^2 texels.
 * Everything that reads the lensmap then reads this one: the warps, blinky_get_lensmap[_packed],
 * blinky_get_display (a plate is displayed when some mapped entry samples it), blinky_mapped_pixels,
 * the tile plan and its queries, blinky_upload_bytes_per_frame, blinky_save_globe and the face-layout
 * checks.  The lens, globe, zoom and rubix settings stay as they are; like a build, the call consumes
 * the lens / globe / zoom changes, so blinky_needs_rebuild is 0 for this size until the next change.
 * An entry without BLINKY_LM_VALID is unmapped whatever its other bits hold and is stored as
 * BLINKY_LM_TINT_NONE << 28, so the map plans and reads back like a build's.  BLINKY_E_INVALID,
 * changing nothing and launching nothing, for a NULL map, width or height <= 0, numplates outside
 * 1..6, platesize <= 0, numplates * platesize^2 above 2^28, or a mapped entry whose index is not below
 * numplates * platesize^2 or whose tint is 6.  A screen wider or taller than 65536 pixels gets no tile
 * plan (the direct-gather kernels warp it).  A graph that captured a warp before the call keeps
 * rendering the map it captured until blinky_release_captures.
 * blinky_set_lensmap reads host memory and also works on host-only contexts (the planner and the
 * queries without a GPU).  blinky_set_lensmap_device reads device memory on `stream` (a cudaStream_t,
 * NULL = the default stream) after the work already there, checks and plans the map on the GPU, and
 * returns once the map is resident: the caller may then reuse d_packed.  BLINKY_E_NODEVICE on a
 * host-only context.  The map itself is copied to the host only when a host-side query needs it. */
int blinky_set_lensmap(blinky_ctx *ctx, int width, int height, int platesize, int numplates, const uint32_t *packed);
int blinky_set_lensmap_device(blinky_ctx *ctx, int width, int height, int platesize, int numplates, const uint32_t *d_packed,
                              void *stream);

/* Ray maps: the lens supplied as data.  A lens is one view ray per screen pixel (lens_inverse,
 * fisheye.c:2084-2124); the globe maps each ray to a plate texel and a rubix tint (:1922-2066).  These
 * calls take the rays and do the globe's half, so a lens that is a table, a calibrated dome or
 * projector warp, a camera model fitted elsewhere or a view turned by head tracking needs no script.
 * rays: width*height float32 triples, row-major, dense: pixel (lx, ly) at rays[3*(ly*width + lx) + k],
 * ly = 0 the top row, in the globe's frame.  Each triple is what lens_inverse returns, narrowed to
 * float and NOT normalised: the library normalises it as the build does (VectorNormalize), and
 * normalising twice is not exact, so a caller that normalises first gets a slightly different map.  A
 * pixel the lens leaves empty is the zero vector (it maps to nothing, as in the reference); NaN and
 * infinite components follow the reference's arithmetic.  The rays go through the current globe: its
 * plates, its globe_plate script if it has one (with the plate slots an earlier globe left, as in a
 * build), and the current f_rubixgrid; the result equals what blinky_build_lensmap makes of a lens
 * returning these rays.  platesize <= 0 means min(width, height), and 6 * platesize^2 must stay below
 * 2^28.  The lens, zoom and blinky_scale are untouched; like a build, the call consumes the lens, globe
 * and zoom changes.  The map is installed as blinky_set_lensmap installs one (every query and warp
 * then reads it; a graph captured before keeps its map until blinky_release_captures).  On failure
 * nothing changes: BLINKY_E_INVALID for NULL or misaligned rays or a bad size, BLINKY_E_STATE without
 * a valid globe, BLINKY_E_SCRIPT when globe_plate raises an error.
 * blinky_set_raymap reads host memory on the worker threads and works on host-only contexts.
 * blinky_set_raymap_device reads d_rays (4-byte aligned device memory) on `stream` (a cudaStream_t,
 * NULL = the default stream) after the work already there, maps and plans on the GPU, and returns once
 * the map is resident: the caller may then reuse d_rays.  Pixels whose globe_plate decision the GPU
 * cannot prove are settled by the interpreter; when that is not possible (globe_plate outside the
 * translatable subset, no NVRTC, too many such pixels) the rays are copied to the host and take the
 * host path.  blinky_build_info says which path ran and how many pixels the interpreter settled.  Not
 * while a stream is capturing.  BLINKY_E_NODEVICE on a host-only context. */
int blinky_set_raymap(blinky_ctx *ctx, int width, int height, int platesize, const float *rays);
int blinky_set_raymap_device(blinky_ctx *ctx, int width, int height, int platesize, const float *d_rays, void *stream);

/* Ray export: the other half of a ray map.  Writes the view rays a width x height build of the current
 * lens evaluates, in the layout blinky_set_raymap reads: float32[height][width][3], dense, ly = 0 the
 * top row.  Pixel (lx, ly) gets lens_inverse((lx - width/2) * scale, -(ly - height/2) * scale), with
 * integer /2 as in the build (fisheye.c:2100-2105) and scale what the current zoom gives for width x
 * height; each component narrowed with static_cast<float> and NOT normalised; (0, 0, 0) where
 * lens_inverse returns nil; NaN and infinities pass through the narrowing.  So for every inverse lens
 * on every globe, with or without a rubix grid, blinky_set_raymap(width, height, platesize, rays) after
 * an export installs the lensmap blinky_build_lensmap(width, height, platesize, ...) installs: the
 * packed map, the display flags, the mapped count and the tile plan.  A head-tracked view exports once,
 * turns the rays each frame (its own kernel) and sets them with blinky_set_raymap_device.  The loaded
 * lens_inverse is evaluated; the lens script is not run again (the purity every threaded or device
 * build assumes).  No globe is needed.  Nothing of the context changes: not the installed lensmap, its
 * plan or generation, blinky_scale, blinky_width/height/platesize, blinky_needs_rebuild or the lens /
 * globe / zoom change flags; blinky_build_info reports the export ("ray export, device: ..." or "ray
 * export, host ...").  On failure the context does not change and the buffer's contents are
 * unspecified: BLINKY_E_INVALID for NULL or misaligned rays or width / height <= 0; BLINKY_E_STATE
 * without a valid lens or for a lens that maps with lens_forward (it has no per-pixel ray);
 * BLINKY_E_ZOOM when the zoom cannot be computed (the build's console message is printed);
 * BLINKY_E_SCRIPT when lens_inverse raises an error or returns anything but three numbers or one nil.
 * blinky_get_raymap writes host memory on the worker threads and works on host-only contexts.
 * blinky_get_raymap_device writes d_rays (4-byte aligned device memory) on `stream` (a cudaStream_t,
 * NULL = the default stream) after the work already there, evaluating the translated lens on the GPU;
 * pixels whose ray the GPU cannot prove equal to the interpreter's are evaluated by the interpreter and
 * written in stream order.  When that is not possible (a lens outside the translatable subset, no
 * NVRTC, too many such pixels) the rays are made on the host and copied to d_rays in stream order.  It
 * returns once d_rays holds the complete field.  BLINKY_E_STATE while `stream` is capturing a graph
 * (nothing is launched); BLINKY_E_NODEVICE on a host-only context. */
int blinky_get_raymap(blinky_ctx *ctx, int width, int height, float *rays);
int blinky_get_raymap_device(blinky_ctx *ctx, int width, int height, float *d_rays, void *stream);

/* Ray export of a forward lens (DESIGN section 3h): the view rays of any lens whose lens_forward is a
 * function, whatever its `map`, so that lenses without lens_inverse (sinusoidal, winkel1, ...) can feed
 * the ray warps too.  Same layout as blinky_get_raymap: float32[height][width][3], dense, ly = 0 the top
 * row.  The rays come from the forward build of the current lens and globe at width x height on plates
 * of platesize texels (platesize <= 0: min(width, height), as blinky_build_lensmap; 6 * platesize^2 must
 * stay below 2^28, so a 4K export wants an explicit platesize), at the scale the current zoom gives for
 * width x height.  That build's grid points, stale slots, texel owners (plate argmax or globe_plate) and
 * maxdiff guard apply, and:
 *   - a pixel is non-zero exactly when that build's lensmap maps it; the others are (0, 0, 0);
 *   - the texel (P, px, py) that last wrote the pixel drew it with a quad of integer screen corners
 *     tl, tr (grid row py, v = (py - 1/2) / ps) and bl, br (row py + 1), grid point i at u = (i - 1/2) / ps;
 *   - measured in half pixels (a corner c came from (int)(x / scale + width/2) and sits at 2c + 1, pixel
 *     X at 2X), the pixel's (s, t) in the quad (tl = (0,0), tr = (1,0), br = (1,1), bl = (0,1)) comes
 *     from the first non-degenerate triangle of A = (tl, tr, br), B = (tl, br, bl) that contains it
 *     (boundary included), by exact integer areas and one double division each; when neither contains it,
 *     from the first non-degenerate one, clamped to [0, 1]; when both are degenerate, or a corner lies
 *     further than the raster's maxdiff (20) from tl, s = t = 1/2;
 *   - the ray is plate_uv_to_ray(P, ((px - 1/2) + s) / ps, ((py - 1/2) + t) / ps), normalised.
 * It is a function of the build's integer state, so the host and the GPU write the same bits.  Each
 * corner is within half a pixel of where lens_forward puts its grid point, so away from seams a ray
 * projects back to within about a pixel of its pixel (DESIGN 3h gives the measured bounds).  Nothing is
 * printed (no "> maxdiff" lines) and the context does not change, as for blinky_get_raymap;
 * blinky_build_info reports the export ("ray export (forward), device: ..." or "... host ...").
 * blinky_get_raymap keeps refusing lenses that map with lens_forward.  On failure the buffer's contents
 * are unspecified: BLINKY_E_INVALID for NULL or misaligned rays, width / height <= 0 or a platesize
 * beyond the limit; BLINKY_E_STATE without a valid lens, a lens_forward function or a valid globe;
 * BLINKY_E_ZOOM when the zoom cannot be computed; BLINKY_E_SCRIPT when lens_forward or globe_plate fails.
 * blinky_get_raymap_forward runs the serial forward builder on the host and works on host-only contexts.
 * blinky_get_raymap_forward_device evaluates the grid points on the GPU (the unit blinky_build_lensmap
 * compiles for this lens), settles the points it cannot prove on the host, and rasterises and writes
 * d_rays (4-byte aligned device memory) on `stream` (a cudaStream_t, NULL = the default stream) after the
 * work already there; when that is not possible (no NVRTC, a lens outside the translatable subset) the
 * host path runs and the field is copied in stream order.  It returns once d_rays holds the field.
 * BLINKY_E_STATE while `stream` is capturing a graph (nothing is launched); BLINKY_E_NODEVICE on a
 * host-only context. */
int blinky_get_raymap_forward(blinky_ctx *ctx, int width, int height, int platesize, float *rays);
int blinky_get_raymap_forward_device(blinky_ctx *ctx, int width, int height, int platesize, float *d_rays, void *stream);

/* ---- state queries ------------------------------------------------------ */
int blinky_fisheye_enabled(blinky_ctx *ctx);          /* fisheye_enabled, :293 */
int blinky_lens_valid(blinky_ctx *ctx);
int blinky_globe_valid(blinky_ctx *ctx);
const char *blinky_lens_name(blinky_ctx *ctx);
const char *blinky_globe_name(blinky_ctx *ctx);
const char *blinky_lens_onload(blinky_ctx *ctx);      /* "" when nil */
int blinky_map_type(blinky_ctx *ctx);
int blinky_zoom_type(blinky_ctx *ctx);
int blinky_zoom_fov(blinky_ctx *ctx);
int blinky_max_fov(blinky_ctx *ctx);
int blinky_max_vfov(blinky_ctx *ctx);
double blinky_lens_width(blinky_ctx *ctx);
double blinky_lens_height(blinky_ctx *ctx);
double blinky_scale(blinky_ctx *ctx);                 /* lens.scale after a build */
int blinky_rubix_enabled(blinky_ctx *ctx);
int blinky_numplates(blinky_ctx *ctx);
int blinky_platesize(blinky_ctx *ctx);
int blinky_width(blinky_ctx *ctx);
int blinky_height(blinky_ctx *ctx);
/* per plate: forward[3] right[3] up[3] fov dist as 11 floats; returns numplates */
int blinky_get_plates(blinky_ctx *ctx, float *out, int max_plates);
/* globe.plates[i].display after a build (:1976): which plates the lens uses */
int blinky_get_display(blinky_ctx *ctx, int out[BLINKY_MAX_PLATES]);
double blinky_plate_fov(blinky_ctx *ctx, int plate);  /* radians: fisheye_plate_fov source, :769 */
/* six 256-entry tint LUTs (globe.plates[i].palette) */
int blinky_get_palmaps(blinky_ctx *ctx, uint8_t out[BLINKY_MAX_PLATES * 256]);
/* lensmap in the reference's terms: idx = pointer - globe.pixels or -1; tint 0..5 or 255 */
int blinky_get_lensmap(blinky_ctx *ctx, int32_t *idx, uint8_t *tint);
/* the packed 32-bit entries the kernels read */
int blinky_get_lensmap_packed(blinky_ctx *ctx, uint32_t *out);
int64_t blinky_mapped_pixels(blinky_ctx *ctx);        /* M in the 5*W*H + M byte count */
/* direct script probes (LUAtoC_lens_inverse/_forward before float narrowing):
 * return 1 = values, 0 = nil, negative = error */
int blinky_lens_inverse(blinky_ctx *ctx, double x, double y, double ray_out[3]);
int blinky_lens_forward(blinky_ctx *ctx, double rx, double ry, double rz, double *x, double *y);
/* the globe's globe_plate(x, y, z) as the lensmap build reads it (ray_to_plate_index,
 * fisheye.c:2027-2033): 1 = a plate (*plate = the last value returned, converted like
 * lua_tointeger: (int)(ptrdiff_t)d), 0 = no value, nil or not a number (*plate = -1),
 * negative = error (-2: the globe has no globe_plate, -3: script error) */
int blinky_globe_plate(blinky_ctx *ctx, double x, double y, double z, int *plate);
/* The current lens function translated to C++ / CUDA C++ — what the device lensmap builder
 * compiles (SURVEY 8f).  flavour: bit 0 = CUDA (else plain C++), bit 1 = lens_forward (else
 * lens_inverse), bit 2 = append the fixed kernel (the per-pixel / per-grid-point tail) and, when
 * the globe has a globe_plate script, translate it into the same unit — with bits 0 and 2 this is
 * exactly what NVRTC is given.  bit 3 = the globe's globe_plate translated alone (bit 0 still picks
 * CUDA; bits 1 and 2 are ignored).  bit 4 = the ray-map unit of blinky_set_raymap_device: the globe's
 * globe_plate translated alone (nothing for globes without one) and the ray-map kernel; with bit 0
 * this is exactly what NVRTC is given (bits 1 to 3 are ignored).  bit 5 = the ray-export unit of
 * blinky_get_raymap_device: lens_inverse translated alone and the ray-export kernel; with bit 0 this is
 * exactly what NVRTC is given (bits 1 to 4 are ignored).  Returns the bytes needed (excluding NUL), or BLINKY_E_SCRIPT
 * when the lens (or globe_plate) is missing or outside the translatable subset (reason:
 * blinky_last_error). */
int blinky_lens_source(blinky_ctx *ctx, int flavour, char *buf, size_t bufsize);
/* F_WriteConfig text; returns bytes needed (excluding NUL) */
int blinky_write_config(blinky_ctx *ctx, char *buf, size_t bufsize);

/* f_saveglobe (fisheye.c:1120-1136, 1396-1486): the console command arms a request;
 * the frame driver asks blinky_saveglobe_pending() after rendering the plates and then
 * passes them to blinky_save_globe(), which writes <directory>/<name><i>.pcx per plate
 * (the reference's COM_WriteFile target is com_gamedir) and prints "Wrote ...". */
int blinky_saveglobe_pending(blinky_ctx *ctx);
int blinky_save_globe(blinky_ctx *ctx, const uint8_t *faces_host, const char *directory);

/* ---- hot path ("RenderLensMap") — GPU only ------------------------------- */
int blinky_set_kernel(blinky_ctx *ctx, int kernel_variant);
/* Frame shown where the lens maps nothing (what Draw_TileClear left in
 * vid.buffer, :802).  [height][width] bytes, NULL = all zero.  Uploaded once. */
int blinky_set_background(blinky_ctx *ctx, const uint8_t *background_host);

/* Face layout: where the plates sit in each frame of the faces the warps read, for hosts that render
 * plates into surfaces of their own (a 3x2 atlas, viewports of one render target, a surface with a
 * padded row pitch) and warp straight from there instead of repacking.  Each frame is a surface with
 * rows of `rowbytes` bytes; plate i starts at byte x = origins[2i], row y = origins[2i+1], so texel
 * (px, py) of plate i in frame f is at
 *     faces + f * face_stride + (y + py) * rowbytes + x + px.
 * rowbytes = 0 (origins ignored) restores the dense nframes x [numplates][ps][ps] faces, the default.
 * Context state read when a warp is enqueued, like blinky_set_background: it applies to
 * blinky_warp_device, _rgba, _view, _view_rgba, _view_rgba_tables, blinky_warp_host (the sampled
 * rectangle of each plate is copied out of the surface), blinky_shard_warp_gather and blinky_save_globe.
 * A captured warp keeps the layout in effect at capture; a later call does not change its replays.
 * Works on host-only contexts (for blinky_save_globe).  BLINKY_E_INVALID, changing nothing, for
 * rowbytes < 0, origins NULL with rowbytes > 0, nplates outside 1..6, or a negative coordinate.
 * The plate size and the plates a lens samples change with every build, so each warp checks the
 * layout against the current lensmap and fails with BLINKY_E_INVALID, launching nothing, when a plate
 * the lensmap samples has no origin, a plate's x + ps exceeds rowbytes, or nframes > 1 and
 * face_stride is less than the surface, max(y + ps) * rowbytes.  The ring kernel reads a layout
 * through TMA, which needs rowbytes and every x origin to be multiples of 16 (and the faces 16-byte
 * aligned, as for dense faces); any other layout is warped by the direct-gather kernel. */
int blinky_set_face_layout(blinky_ctx *ctx, int rowbytes, const int32_t *origins, int nplates);

/* Device-resident batch: d_faces -> d_out on `stream` (a cudaStream_t; NULL is
 * CUDA's default stream).  d_faces: nframes x [numplates][ps][ps]
 * bytes, frame stride face_stride bytes; d_out: nframes x [height][width]
 * bytes, stride out_stride.  Asynchronous.  One kernel launch per call. */
int blinky_warp_device(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out, size_t out_stride,
                       int nframes, void *stream);

/* Device-resident batch into a view rectangle of a device framebuffer (scr_vrect, VBUFFER :634).
 * d_screen: nframes screens, frame stride screen_frame_stride bytes, rows of rowbytes bytes; the
 * width x height view starts at pixel (x0, y0).  keep_unmapped != 0: only mapped pixels are written
 * (:2413); otherwise unmapped pixels of the rectangle get the background.  Nothing outside the
 * rectangle is written, and no pixel is read back and rewritten: unmapped pixels are skipped with
 * byte (RGBA: 32-bit) stores, so other writers may fill neighbouring rectangles of the same screen at
 * the same time, from other contexts and streams.  Asynchronous on `stream`, like blinky_warp_device.
 * Fails with BLINKY_E_INVALID, launching nothing, for a NULL buffer, x0 < 0 or y0 < 0,
 * rowbytes < (x0 + width) * bytes per pixel, or nframes > 1 with
 * screen_frame_stride < (y0 + height) * rowbytes.  Views whose width, origin, rowbytes and frame
 * stride are multiples of 4 pixels take the fast kernels; any other view is warped pixel by pixel.
 *
 * CUDA graphs.  blinky_warp_device, blinky_warp_device_rgba, blinky_warp_device_view,
 * blinky_warp_device_view_rgba and blinky_warp_device_view_rgba_tables may be called while `stream` is
 * capturing (cudaStreamBeginCapture in any mode, torch.cuda.graph): they then allocate, copy and
 * synchronise nothing, and the launches land in the graph.  A replay, on any stream and beside eager
 * warps and other graphs of the same context, reads
 *   - the lensmap and tile plan of the capture (a later blinky_build_lensmap does not invalidate the
 *     graph: the buffers it would free are kept for the graph);
 *   - the faces, output and per-frame table pointers given at capture, with whatever they hold when the
 *     replay runs (so a cudaMemcpyAsync into the tables on the replay's stream changes the palette);
 *   - the background, rubix LUTs and RGBA table as they are when the replay runs (after a rebuild to
 *     another view size: the background of the captured size);
 *   - the face layout (blinky_set_face_layout) that was in effect at capture.
 * Each captured launch of the ring kernel takes one of 4096 work counters; when none is left the call
 * fails with BLINKY_E_STATE and launches nothing.  blinky_warp_host, blinky_shard_warp_gather,
 * blinky_build_lensmap, blinky_set_lensmap, blinky_set_lensmap_device, blinky_set_background and
 * blinky_set_rgba_table must not be called while a stream is capturing. */
int blinky_warp_device_view(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_screen,
                            size_t screen_frame_stride, int rowbytes, int x0, int y0, int nframes,
                            int keep_unmapped, void *stream);
/* States that no graph which captured a warp of this context will run again (destroy those graphs
 * first, or keep them and never launch them): synchronises the device, frees the lensmap buffers
 * rebuilds kept for graphs, and returns every capture work counter.  Call it after retiring a set of
 * graphs, e.g. when a lens change makes them stale.  BLINKY_E_INVALID, changing nothing, while a capture
 * that holds a warp of this context is still open (it asks each stream such a warp was captured on, so
 * call it before destroying those streams).  blinky_destroy does the same. */
int blinky_release_captures(blinky_ctx *ctx);

/* End to end from HOST buffers: pinned-staged cudaMemcpyAsync of each frame's
 * displayed plates, the warp, and the copy back, software-pipelined over
 * internal streams.  faces_host: nframes x [numplates][ps][ps].  dst_host: nframes
 * screens of dst_rowbytes pitch; the view rectangle starts at (x0,y0) inside
 * each (scr_vrect, VBUFFER macro :634).  If keep_unmapped != 0 only mapped
 * pixels are written into dst (exact reference semantics, :2413); otherwise
 * unmapped pixels receive the background set above.  Synchronous. */
int blinky_warp_host(blinky_ctx *ctx, const uint8_t *faces_host, size_t face_stride, uint8_t *dst_host,
                     size_t dst_frame_stride, int dst_rowbytes, int x0, int y0, int nframes, int keep_unmapped);

/* bytes blinky_warp_host copies host->device per frame for the current lensmap: for
 * every plate the lens shows, the texel rectangle it samples */
int64_t blinky_upload_bytes_per_frame(blinky_ctx *ctx);

/* pinned host memory helpers for callers that want zero staging copies */
int blinky_alloc_pinned(blinky_ctx *ctx, size_t bytes, void **out);
int blinky_free_pinned(blinky_ctx *ctx, void *ptr);
int blinky_sync(blinky_ctx *ctx);

/* ---- peer memory: fused warp + gather over NVLink ------------------------------
 * The kernels write through whatever device-accessible pointer d_out is.  To fuse the
 * reference topology's final gather into the warp, rank 0 allocates the gather buffer,
 * exports it, every other rank (one process per GPU) opens it and passes
 * `peer_base + its frame offset` as d_out: finished pixels then travel to rank 0 as
 * NVLink stores issued by the warp kernel itself, no separate collective.
 * handle: 64 opaque bytes (cudaIpcMemHandle_t), moved between processes by the caller. */
int blinky_alloc_device(blinky_ctx *ctx, size_t bytes, void **out);
int blinky_free_device(blinky_ctx *ctx, void *ptr);
int blinky_ipc_export(blinky_ctx *ctx, void *device_ptr, unsigned char handle[64]);
int blinky_ipc_open(blinky_ctx *ctx, const unsigned char handle[64], void **peer_ptr);
int blinky_ipc_close(blinky_ctx *ctx, void *peer_ptr);

/* ---- sharded batches: frames over N GPUs, finished frames gathered on rank 0 -----------------
 * One process per GPU, one context per process.  A batch of total_frames independent frames is cut
 * into contiguous blocks (blinky_shard_range, sizes differ by at most one); every rank builds the same
 * lensmap and warps its own block; there is NO collective on the data path.  The reference topology's
 * last step — finished frames reach the one display (the reference writes vid.buffer,
 * engine/NQ/fisheye.c:802-803, 2406-2424) — is a gather to rank 0, done chunk by chunk so that the
 * transfer of chunk k overlaps the warp of chunk k+1 (a compute and a communication stream per rank).
 *   BLINKY_GATHER_NCCL        ncclSend / ncclRecv of finished chunks (NCCL only for the final gather)
 *   BLINKY_GATHER_PEER_COPY   copy engines push finished chunks into rank 0's buffer (CUDA-IPC peer memory over NVLink)
 *   BLINKY_GATHER_PEER_STORE  the warp kernels store straight into rank 0's buffer (fused warp + gather)
 * NCCL is loaded at run time (libnccl.so.2, or the path in BLINKY_NCCL_LIB); the 128-byte id made by
 * blinky_shard_unique_id on one rank is carried to the others by the caller (MPI, a file, torch.distributed ...).
 * Calls marked collective must be made by every rank. */
enum { BLINKY_GATHER_NCCL = 0, BLINKY_GATHER_PEER_COPY = 1, BLINKY_GATHER_PEER_STORE = 2 };
/* pure arithmetic (no context): frames [*first, *first + *count) belong to `rank` */
int blinky_shard_range(int total_frames, int rank, int world, int *first, int *count);
int blinky_shard_unique_id(unsigned char id[128]);
/* collective: joins the group (ncclCommInitRank) */
int blinky_shard_init(blinky_ctx *ctx, int rank, int world, const unsigned char id[128]);
/* collective: rank 0 allocates the gather buffer (total_frames x [height][width] bytes, frame f at
 * f*width*height) and shares it; *root_buffer is that device pointer on rank 0 and NULL elsewhere.
 * Needs a built lensmap.  The buffer lives until the next call or blinky_shard_close. */
int blinky_shard_buffer(blinky_ctx *ctx, int total_frames, void **root_buffer);
/* collective: d_faces = this rank's block of frames (device memory, frame stride face_stride).
 * Stream-ordered: the work starts after what `stream` holds and `stream` then waits for it; on rank 0
 * the gathered batch is complete when `stream` reaches that point. */
int blinky_shard_warp_gather(blinky_ctx *ctx, const void *d_faces, size_t face_stride, int total_frames, int mode,
                             int chunk_frames, void *stream);
int blinky_shard_sync(blinky_ctx *ctx);
int blinky_shard_close(blinky_ctx *ctx);

/* Fused 8-bit -> 32-bit palette expansion (engine/common/vid_sdl.c:539-546,
 * d_8to24table): same warp, output one uint32 per pixel.  table: 256 entries.
 * blinky_set_rgba_table is a blocking host-side replacement of the context's one table (a synchronous
 * copy, outside any stream's order; not while a stream captures).  To change palettes from frame to frame
 * in stream order (V_UpdatePalette's flashes and fades), and per frame within a batch, use
 * blinky_warp_device_view_rgba_tables. */
int blinky_set_rgba_table(blinky_ctx *ctx, const uint32_t table[256]);
int blinky_warp_device_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out_rgba,
                            size_t out_stride, int nframes, void *stream);
/* blinky_warp_device_view with one uint32 per pixel through the blinky_set_rgba_table table: rowbytes
 * and screen_frame_stride in bytes, x0 in pixels.  The view origin, rowbytes and (nframes > 1) the
 * frame stride must be 4-byte aligned, else BLINKY_E_INVALID. */
int blinky_warp_device_view_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_screen_rgba,
                                 size_t screen_frame_stride, int rowbytes, int x0, int y0, int nframes,
                                 int keep_unmapped, void *stream);
/* blinky_warp_device_view_rgba, with frame f expanded through its own 256-entry table at
 * d_tables + f * table_stride bytes instead of the context's blinky_set_rgba_table table.
 * table_stride == 0: one table for every frame.  The tables are device memory, read when the
 * launch runs (stream order: a cudaMemcpyAsync into them earlier on `stream` is seen), so the call
 * is capturable like every blinky_warp_device* call and a replay reads the tables' contents at
 * replay time.  The context's own table is neither read nor changed.  Rubix tints apply before the
 * expansion; without keep_unmapped an unmapped pixel is the background byte through frame f's table.
 * Besides the checks of blinky_warp_device_view_rgba, fails with BLINKY_E_INVALID, launching nothing,
 * when d_tables is NULL or not 16-byte aligned, or table_stride is nonzero and below 1024 or not a
 * multiple of 16. */
int blinky_warp_device_view_rgba_tables(blinky_ctx *ctx, const void *d_faces, size_t face_stride,
                                        void *d_screen_rgba, size_t screen_frame_stride, int rowbytes, int x0,
                                        int y0, int nframes, int keep_unmapped, const uint32_t *d_tables,
                                        size_t table_stride, void *stream);

/* Warp from a ray field turned by a per-frame 3x3 matrix: each pixel's texel is computed on the GPU
 * from its view ray, so a head-tracked look-around needs no lensmap, plan or install per frame.
 * W, H and ps are those of the installed lensmap (blinky_width, blinky_height, blinky_platesize), which
 * also gives the background; without one the call fails with BLINKY_E_STATE.  Frame f reads
 *   - the ray field at d_rays + f * ray_stride bytes: float32[H][W][3] as blinky_set_raymap reads it
 *     (ray_stride 0: one field for every frame);
 *   - the matrix M_f at d_xforms + f * xform_stride bytes: 9 floats, row-major (xform_stride 0: one
 *     matrix for every frame; d_xforms NULL: no turn, the rays are used exactly as read);
 *   - the faces at d_faces + f * face_stride, in the current face layout.  Without one they are dense
 *     [numplates][ps][ps] frames of the GLOBE's numplates (blinky_numplates): after a turn any plate of
 *     the globe may be sampled, not only those of the installed lensmap, so a frame must hold
 *     numplates * ps^2 bytes even when a supplied lensmap has fewer plates.
 * Each pixel's ray (x, y, z) is turned in float32 with round-to-nearest and no fused multiply-add:
 * t_k = (M[k][0]*x + M[k][1]*y) + M[k][2]*z.  Any matrix is accepted, a rotation or not.  The pixel then
 * gets the entry blinky_set_raymap(W, H, ps, t) installs for it through the CURRENT globe (normalised,
 * plate argmax over the globe's plates, lowest index winning ties; an on-grid texel gets no tint), and
 * is written as blinky_warp_device_view writes that entry (RGBA: as
 * blinky_warp_device_view_rgba_tables, with d_tables NULL meaning the blinky_set_rgba_table table):
 * same view rectangle, keep_unmapped, background, f_rubix LUTs and per-frame tables.  In short, frame f
 * equals blinky_set_raymap of the turned field followed by a one-frame view warp.  Nothing outside the
 * view rectangle is written, and no pixel is read back.  The context does not change (lensmap, its
 * plan, blinky_needs_rebuild, display flags, build_info); blinky_launch_count and blinky_last_kernel do.
 * Refusals launch nothing: BLINKY_E_NODEVICE on a host-only context; BLINKY_E_STATE without a valid
 * globe, when the globe picks its plates with a globe_plate script (use blinky_set_raymap_device), or
 * when the installed lensmap's ps is beyond what blinky_set_raymap takes (6 * ps^2 > 0x0FFFFFFF, i.e.
 * ps > 6688, which a supplied lensmap of fewer plates may have);
 * BLINKY_E_INVALID for NULL faces, rays or screen, rays or matrices not 4-byte aligned, a nonzero
 * ray_stride below 12*W*H or not a multiple of 4, a nonzero xform_stride below 36 or not a multiple of
 * 4, more than 65535 frames, any check blinky_warp_device_view[_rgba_tables] makes, and a face layout
 * in which any plate of the globe (not only those the lensmap shows) has no origin or does not fit.
 * Both calls may be captured like blinky_warp_device_view: a replay reads the rays, matrices, tables,
 * faces and screen at the pointers given at capture with their contents at replay time, the globe's
 * plates, rubix grid, f_rubix, face layout and view of the capture, and the background and LUTs as
 * the other warps do; blinky_release_captures covers these graphs too. */
int blinky_warp_device_rays(blinky_ctx *ctx, const void *d_faces, size_t face_stride, const float *d_rays,
                            size_t ray_stride, const float *d_xforms, size_t xform_stride, void *d_screen,
                            size_t screen_frame_stride, int rowbytes, int x0, int y0, int nframes,
                            int keep_unmapped, void *stream);
int blinky_warp_device_rays_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, const float *d_rays,
                                 size_t ray_stride, const float *d_xforms, size_t xform_stride,
                                 void *d_screen_rgba, size_t screen_frame_stride, int rowbytes, int x0, int y0,
                                 int nframes, int keep_unmapped, const uint32_t *d_tables, size_t table_stride,
                                 void *stream);

/* Anti-aliased RGBA warp from a ray field: k x k view rays per pixel (k = factor, 2, 3 or 4),
 * box-filtered.  W, H, ps and the background are the installed lensmap's, as for
 * blinky_warp_device_rays_rgba.  Frame f reads
 *   - the field at d_rays + f * ray_stride bytes, a dense float32[k*H][k*W][3] field (ray_stride 0: one
 *     field for every frame);
 *   - the matrices and faces as blinky_warp_device_rays_rgba reads them;
 *   - the 256-entry table T_f at d_tables + f * table_stride bytes, or the blinky_set_rgba_table table
 *     when d_tables is NULL.
 * Output pixel (x, y) has k^2 samples s = (i, j), 0 <= i, j < k.  Sample s is field pixel
 * (k*x + i, k*y + j), turned by M_f exactly as blinky_warp_device_rays turns a ray, and gets the entry
 * blinky_set_raymap(k*W, k*H, ps, turned field) installs for it through the current globe, with ps the
 * installed lensmap's.  From the entry: byte b_s = the face texel (through the plate's rubix LUT when
 * f_rubix is on and the texel is off the grid) if mapped, else bg[y][x], the OUTPUT pixel's background;
 * colour c_s = T_f[b_s].  Byte n (0..3, little-endian) of the output word is
 * (sum_s byte_n(c_s) + k^2/2) / k^2 in integers (k^2/2 rounds down: 4 for k = 3): round-half-up per
 * channel, alpha averaged like the others.  The average is of the table's bytes as they are (gamma-
 * encoded, as the tables are), not in linear light: so the rule stays a pure integer function of the
 * one-sample warp.  With keep_unmapped a pixel none of whose k^2 samples is mapped is not written, and a
 * partly mapped pixel is written with its unmapped samples taking the background colour.  Nothing
 * outside the view rectangle is written, and no pixel is read back.  Equivalently, frame f is the k x k
 * box average of blinky_warp_device_rays_rgba at k*W x k*H whose background is bg with each byte
 * repeated k x k.
 * Fields: blinky_get_raymap_device(ctx, k*W, k*H, ...) exports the current lens at the k-fold size.
 * Sample i of pixel x then lies at about (x + i/k - W/2) * scale, so the box spans [x, x + (k-1)/k] and
 * sits less than half a pixel off the one-sample warp's (x - W/2) * scale; a caller wanting centred
 * boxes supplies its own field.
 * Refuses everything blinky_warp_device_rays_rgba refuses, with the same codes, and launches nothing
 * when it does; BLINKY_E_INVALID also when factor is not 2, 3 or 4 (k = 1 is
 * blinky_warp_device_rays_rgba), a nonzero ray_stride is below 12*k^2*W*H, or k^2*W*H is beyond the
 * kernel's 31-bit pixel index (2^31 - 1).  Capturable like blinky_warp_device_rays_rgba, on the same
 * terms; the context does not change, blinky_launch_count and blinky_last_kernel do. */
int blinky_warp_device_rays_supersampled(blinky_ctx *ctx, const void *d_faces, size_t face_stride,
                                         const float *d_rays, size_t ray_stride, const float *d_xforms,
                                         size_t xform_stride, int factor, void *d_screen_rgba,
                                         size_t screen_frame_stride, int rowbytes, int x0, int y0, int nframes,
                                         int keep_unmapped, const uint32_t *d_tables, size_t table_stride,
                                         void *stream);

/* Bilinear-filtered RGBA warp from a ray field, alone (factor k = 1) or under k x k supersampling
 * (k = 2, 3 or 4).  Same arguments as blinky_warp_device_rays_supersampled: W, H, ps and the background
 * are the installed lensmap's, and the field (float32[k*H][k*W][3]), matrices, faces, tables, view
 * rectangle, keep_unmapped and face layout are read as that call reads them.  Sample s of output pixel
 * (x, y) is field pixel (k*x + i, k*y + j), turned by M_f exactly as blinky_warp_device_rays turns a ray.
 *   - Mapping: the sample is mapped exactly when blinky_set_raymap maps the turned ray, on the same
 *     plate P, with u, v the plate coordinates (in double) whose truncation to u*ps, v*ps is its texel.
 *   - Position, one IEEE double operation each: sx = u*ps - 0.5, sy = v*ps - 0.5; x0 = floor(sx),
 *     y0 = floor(sy); wx = (int)((sx - x0) * 256), wy = (int)((sy - y0) * 256), each in 0..255.  The
 *     taps are (x0 | x0+1, y0 | y0+1), each coordinate clamped to [0, ps-1] on plate P: no filtering
 *     across plate seams, and no read outside the plate's ps x ps texels.
 *   - Texel colour: C(tx, ty) = T_f[b'] with b the face byte of (P, tx, ty), b' = LUT_P[b] when f_rubix
 *     is on and texel (tx, ty) is off the rubix grid, else b' = b: the colour
 *     blinky_warp_device_rays_rgba draws for a ray that lands on that texel (grid lines are filtered
 *     like the rest of the image).
 *   - Blend, per byte n (alpha included), in integers: ((C00*(256-wx) + C10*wx)*(256-wy) +
 *     (C01*(256-wx) + C11*wx)*wy + 32768) >> 16, with Cab the tap (x0+a, y0+b).  The weights sum to
 *     65536: a texel centre gives C00 exactly, and a region of one colour stays that colour.  The blend
 *     is of the tables' gamma-encoded bytes, as the supersampled average is.
 *   - An unmapped sample's colour is T_f[bg[y][x]], the output pixel's background.
 * The k^2 sample colours are averaged per byte as (sum + k^2/2) / k^2 (k = 1: the sample's colour).  With
 * keep_unmapped a pixel none of whose samples is mapped is not written.  Equivalently, frame f is the
 * k x k box average of this warp at k = 1 over k*W x k*H, whose background is bg with each byte repeated
 * k x k; at k = 1 with keep_unmapped it writes exactly the pixels blinky_warp_device_rays_rgba writes.
 * There is no 8-bit form: palette indices cannot be blended.
 * Sample positions: an exported field (blinky_get_raymap_device at k*W x k*H) places the samples as
 * blinky_warp_device_rays_supersampled describes.
 * Refuses everything blinky_warp_device_rays_supersampled refuses, with the same codes, and launches
 * nothing when it does; BLINKY_E_INVALID for a factor that is not 1, 2, 3 or 4, and for k^2*W*H beyond
 * the kernel's 31-bit pixel index (2^31 - 1) at every factor, 1 included.  Capturable like
 * blinky_warp_device_rays_rgba, on the same terms; the context does not change, blinky_launch_count
 * and blinky_last_kernel do. */
int blinky_warp_device_rays_bilinear(blinky_ctx *ctx, const void *d_faces, size_t face_stride,
                                     const float *d_rays, size_t ray_stride, const float *d_xforms,
                                     size_t xform_stride, int factor, void *d_screen_rgba,
                                     size_t screen_frame_stride, int rowbytes, int x0, int y0, int nframes,
                                     int keep_unmapped, const uint32_t *d_tables, size_t table_stride,
                                     void *stream);

/* Bytes of one frame's RGBA mip pyramid for blinky_warp_device_rays_trilinear (B below): the installed
 * lensmap's plate size ps and every plate of the current globe.  BLINKY_E_STATE with no lensmap, no
 * valid globe, or ps beyond the ray warps' limit (6688); BLINKY_E_NODEVICE on a host-only context.  The
 * context does not change. */
int blinky_ray_pyramid_bytes(blinky_ctx *ctx, size_t *bytes);

/* Trilinear-filtered (mip-mapped) RGBA warp from a ray field: one sample per pixel, from the two levels of
 * a per-frame mip pyramid around the pixel's footprint, so a view that minifies the plates stays steady
 * as it moves.  W, H, ps and the background are the installed lensmap's; the field (float32[H][W][3]),
 * matrices, faces, face layout, tables, view rectangle and keep_unmapped are read as
 * blinky_warp_device_rays_bilinear reads them at factor 1.
 *   1. Pyramid, per frame, of every plate P of the globe: s_0 = ps, s_L = (s_{L-1} + 1) >> 1 down to
 *      s_Lmax = 1 (ps = 1: Lmax = 0; 97: 7; 2048: 11).  C_0(P, x, y) = T_f[b'], the texel colour of
 *      blinky_warp_device_rays_bilinear.  Level L >= 1, per byte, alpha included:
 *      C_L(x, y) = (sum over i, j in {0, 1} of C_{L-1}(min(2x+i, s_{L-1}-1), min(2y+j, s_{L-1}-1)) + 2) >> 2.
 *      Levels 1..Lmax are written as uint32 RGBA words at d_scratch + f*B (B = blinky_ray_pyramid_bytes):
 *      level-major, then plate 0..numplates-1, then rows [s_L][s_L]; level L's plate 0 starts
 *      4 * numplates * (s_1^2 + ... + s_{L-1}^2) bytes in, and B is the total rounded up to 256.  Level 0
 *      is never stored: it is the faces.
 *   2. Footprint: the pixel's ray r (field pixel (x, y) turned by M_f) is mapped on plate P exactly as
 *      blinky_warp_device_rays_bilinear maps it, with plate coordinates (u, v); unmapped, the pixel is
 *      T_f[bg[y][x]].  The projection of a normalised ray n onto P: x, y, z the float dot products with
 *      P's right, up and forward, widened to double; usable iff z > 0; then q = uv_dist_P * ps / z,
 *      a = x*q, b = -y*q (double, one IEEE operation each).  r's own projection unusable: rho^2 = 0.
 *      Otherwise the x axis uses field pixel (x+1, y) when it exists and its turned, normalised ray
 *      projects usably onto P, else (x-1, y) on the same terms, else it gives 0; the y axis likewise with
 *      (x, y+1) and (x, y-1).  An axis gives da*da + db*db (the differences from r's (a, b)); rho^2 is
 *      the x axis's value, replaced by the y axis's when that is greater.  rho = sqrt(rho^2), correctly
 *      rounded.
 *   3. Level and weight, by comparisons: L the largest L <= Lmax with 2^L <= rho (0 when rho < 1 or NaN);
 *      w = (int)((rho * 2^-L - 1) * 256) when 1 <= rho and L < Lmax, else 0.
 *   4. Colour: C_L at (u, v) is blinky_warp_device_rays_bilinear's blend on level L's grid: sx =
 *      u*s_L - 0.5, x0 = floor(sx), wx = (int)((sx - x0)*256), likewise y, taps clamped to [0, s_L-1]
 *      on plate P (level 0: exactly that call's colour).  The output is C_Lmax when L = Lmax, else per
 *      byte (C_L*(256-w) + C_{L+1}*w + 128) >> 8.
 *   5. With keep_unmapped the pixels blinky_warp_device_rays_rgba skips are skipped.
 * Where rho < 1 at every pixel the output equals blinky_warp_device_rays_bilinear at factor 1.  The
 * scratch is the caller's: nothing is allocated, copied or synchronised, and the pyramid bytes are left
 * in it.  The call adds Lmax + 1 to blinky_launch_count (one launch per pyramid level 1..Lmax, then the
 * warp); blinky_last_kernel names the warp kernel.
 * Refuses everything blinky_warp_device_rays_bilinear refuses at factor 1, with the same codes, and
 * launches nothing when it does; also BLINKY_E_INVALID for a NULL d_scratch while B > 0, a d_scratch
 * that is not 16-byte aligned, and scratch_bytes < nframes * B.  Capturable like
 * blinky_warp_device_rays_rgba, on the same terms; the context does not change. */
int blinky_warp_device_rays_trilinear(blinky_ctx *ctx, const void *d_faces, size_t face_stride,
                                      const float *d_rays, size_t ray_stride, const float *d_xforms,
                                      size_t xform_stride, void *d_screen_rgba, size_t screen_frame_stride,
                                      int rowbytes, int x0, int y0, int nframes, int keep_unmapped,
                                      const uint32_t *d_tables, size_t table_stride, void *d_scratch,
                                      size_t scratch_bytes, void *stream);

/* one-line description of how the current lensmap was tiled for the TMA kernel
 * (tile counts per class, staged bytes per pixel); "" before a build */
const char *blinky_plan_summary(blinky_ctx *ctx);
/* The tile plan the kernels read (DESIGN.md section 3): 16-byte tile descriptors
 * {u32 entry_offset; i16 box_x, box_y; u8 plate (bits 0-2) | tile tint << 3 (0-5, 7 = no pixel tinted),
 * type (0 empty, 1 box, 2 gather, 3 box fully mapped), box_w/16, box_h/8; u16 px, py} — the upper six bits of
 * `type` are the index of the box shape (one TMA descriptor per shape, at most 64) — ordered BOX tiles, GATHER
 * tiles, EMPTY tiles, and the entry blocks in the same order, fixed sizes: BOX 2176 bytes = [4][32 lanes][8]
 * uint16 {bit 15 valid, bits 0-13 offset inside the box} in the ring kernel's lane order (lane l, entry i ->
 * tile row (l>>3) + 4*(i>>2), column 4*(l&7) + (i&3)) followed by [32 lanes] uint32 tint flags (bit i: the
 * lane's pixel i carries the tile's tint; tiles whose tinted pixels disagree are GATHER tiles); GATHER 4096
 * bytes = [32][32] packed 32-bit lensmap entries.  Pass NULL buffers to query the sizes.  Works on CPU-only contexts;
 * the tests interpret the plan on the CPU to pin this layout (tests/test_tile_plan.py). */
int blinky_get_tile_plan(blinky_ctx *ctx, void *tiles_out, size_t tiles_cap, void *entries_out, size_t entries_cap, size_t *ntiles,
                         size_t *entry_bytes);
/* FNV-1a digest of the tile table + entry blocks planned on `threads` host threads (the plan
 * must not depend on the thread count; used by the tests) */
uint64_t blinky_plan_digest(blinky_ctx *ctx, int threads);
/* number of kernel launches issued by this context so far (launches captured into a graph count once,
 * at capture; replays do not count) */
int64_t blinky_launch_count(blinky_ctx *ctx);
/* last warp kernel's name and launch geometry, for reports (a captured launch included) */
const char *blinky_last_kernel(blinky_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* BLINKY_B200_H */
