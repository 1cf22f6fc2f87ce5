/* TEST INFRASTRUCTURE — parity oracle, not part of the product.
 *
 * Plain-C restatement of the reference's lens-warp path
 * (the reference's engine/NQ/fisheye.c), one function per reference function,
 * each citing the lines it follows.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this library; the
 * product (blinky_b200/) never links, imports or executes anything in oracle/.
 *
 * Parity status: PINNED.  The reference has no tests or golden vectors of its
 * own (SURVEY.md section 4), so this restatement is pinned against the
 * reference ITSELF: oracle/_ref/libblinky_ref.so is the unmodified fisheye.c
 * compiled from the original project, and tests/test_oracle_vs_ref.py requires
 * bit-identical lensmaps, tint maps, palette LUTs and rendered frames from
 * both on every shipped globe x lens combination; tests/golden/ holds vectors
 * generated from _ref by tests/golden/make_golden.py for boxes without
 * the original project.
 *
 * The one part of the path that is NOT in the original project is the Lua 5.2 VM
 * (external liblua, engine/Makefile:834-841, BUILDING.md:19-27; no pinned patch
 * version, absent from the image).  Lens functions enter this oracle as C
 * callbacks; oracle_lenses.c holds literal C transcriptions of the BASELINE
 * lens scripts (doubles + libm, exactly what a Lua 5.2 VM executes), which is
 * what pins the product's own Lua-subset evaluator.
 */
#ifndef BLINKY_ORACLE_H
#define BLINKY_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_MAX_PLATES 6 /* fisheye.c:352 */

/* return conventions follow LUAtoC_lens_inverse / _forward (fisheye.c:1545-1632):
 *  1 = values returned, 0 = script returned nil (skip), -1 = error (abort build) */
typedef int (*orc_inverse_fn)(double x, double y, double ray_out[3], void *ud);
typedef int (*orc_forward_fn)(double rx, double ry, double rz, double *x, double *y, void *ud);
/* LUAtoC_globe_plate (fisheye.c:1634-1651): 1 = plate written, 0 = not a number */
typedef int (*orc_globe_plate_fn)(double rx, double ry, double rz, int *plate, void *ud);

typedef struct {
    float forward[3], right[3], up[3]; /* vec3_t = float[3] (mathlib.h:30-31) */
    float fov, dist;                   /* vec_t (fisheye.c:357-358) */
    int display;
} orc_plate;

typedef struct {
    int numplates;
    int platesize;
    orc_plate plates[ORC_MAX_PLATES];
    orc_globe_plate_fn plate_fn; /* NULL = nearest plate by dot product */
    void *plate_ud;
} orc_globe;

typedef struct {
    int numcells;       /* rubix.numcells (int) */
    double cell_size;   /* rubix.cell_size */
    double pad_size;    /* rubix.pad_size */
} orc_rubix;

enum { ORC_ZOOM_NONE = 0, ORC_ZOOM_FOV, ORC_ZOOM_VFOV, ORC_ZOOM_COVER, ORC_ZOOM_CONTAIN };
enum { ORC_MAP_NONE = 0, ORC_MAP_INVERSE, ORC_MAP_FORWARD };

typedef struct {
    int width_px, height_px;
    double scale;
    int32_t *idx;   /* [H][W]: plate*ps*ps + py*ps + px, or -1 (NULL pointer in the reference) */
    uint8_t *tint;  /* [H][W]: plate index or 255 */
} orc_lensmap;

/* --- globe ------------------------------------------------------------- */
/* one plate exactly as LUA_load_globe stores it (fisheye.c:1809-1868) */
void orc_globe_set_plate(orc_globe *g, int i, const double forward[3], const double up[3], double fov_degrees);

/* --- pure converters (fisheye.c:1184-1214) and their Lua-visible wrappers
 *     (fisheye.c:1494-1537), which round through float32 ------------------ */
void orc_latlon_to_ray(double lat, double lon, float ray[3]);
void orc_ray_to_latlon(const float ray[3], double *lat, double *lon);
void orc_plate_uv_to_ray(const orc_globe *g, int plate, double u, double v, float ray[3]);
void orc_lua_latlon_to_ray(double lat, double lon, double out[3]);
void orc_lua_ray_to_latlon(double rx, double ry, double rz, double *lat, double *lon);
int orc_lua_plate_to_ray(const orc_globe *g, double plate, double u, double v, double out[3]);

/* --- zoom (fisheye.c:1293-1386) ---------------------------------------- */
/* returns 1 and writes *scale on success, 0 on any of the reference's failure exits */
int orc_calc_zoom(int zoom_type, int fov, int max_fov, int max_vfov, double lens_width, double lens_height,
                  int width_px, int height_px, orc_forward_fn fwd, void *ud, double *scale);

/* --- lensmap build ------------------------------------------------------ */
/* caller provides idx/tint arrays; they are cleared to -1 / 255 first
 * (fisheye.c:731-732).  Returns 0 = complete, -1 = aborted by a lens error. */
int orc_build_inverse(orc_globe *g, const orc_rubix *rubix, orc_lensmap *lm, orc_inverse_fn inv, void *ud);
int orc_build_forward(orc_globe *g, const orc_rubix *rubix, orc_lensmap *lm, orc_forward_fn fwd, void *ud);

/* --- rubix palette (fisheye.c:835-908) ---------------------------------- */
void orc_create_palmap(const uint8_t palette[768], uint8_t out[ORC_MAX_PLATES][256]);

/* --- the hot loop (fisheye.c:2406-2424) --------------------------------- */
/* vbuf is the screen buffer (vid.buffer); only mapped pixels are written. */
void orc_render_lensmap(const orc_lensmap *lm, const uint8_t *faces, const uint8_t palmaps[ORC_MAX_PLATES][256],
                        int rubix_enabled, uint8_t *vbuf, int rowbytes, int vrect_x, int vrect_y);
/* same loop, rows split over OpenMP threads (the "all host cores" CPU baseline) */
void orc_render_lensmap_omp(const orc_lensmap *lm, const uint8_t *faces, const uint8_t palmaps[ORC_MAX_PLATES][256],
                            int rubix_enabled, uint8_t *vbuf, int rowbytes, int vrect_x, int vrect_y, int threads);
int orc_max_threads(void);
double orc_time_render(const orc_lensmap *lm, const uint8_t *faces, const uint8_t palmaps[ORC_MAX_PLATES][256],
                       int rubix_enabled, uint8_t *vbuf, int rowbytes, int threads, int reps, double *total_seconds);

/* --- C transcriptions of shipped scripts (oracle_lenses.c) -------------- */
/* name: "panini","stereographic","equirect","hammer","fisheye1","fisheye2",
 * "quincuncial","rectilinear","cylinder","mercator".  Returns 0 if unknown. */
typedef struct {
    const char *name;
    orc_inverse_fn inverse;   /* may be NULL */
    orc_forward_fn forward;   /* may be NULL */
    int max_fov, max_vfov;    /* 0 when the script leaves them nil */
    double lens_width, lens_height; /* 0 when nil */
    const char *onload;
} orc_lens_def;
int orc_find_lens(const char *name, orc_lens_def *out);
/* lenses/debug.lua sizes itself from the globe's plate count and needs the globe as `ud` of its inverse */
int orc_debug_lens(int numplates, orc_lens_def *out);
/* name: "cube","trism","tetra","cube_edge","cube_corner","fast" */
int orc_load_globe(const char *name, orc_globe *g);

#ifdef __cplusplus
}
#endif
#endif
