/* TEST INFRASTRUCTURE — not part of the product.
 *
 * Headless harness around the UNMODIFIED reference fisheye layer.  The
 * reference source is pulled in where it lies (`#include "fisheye.c"` resolves
 * through -Ithe reference's engine/NQ, see ../Makefile); nothing is copied into
 * this repository.  Including it in this translation unit gives the harness
 * access to the file-static `lens`, `globe`, `zoom`, `rubix` structures
 * (engine/NQ/fisheye.c:334-528) so the lensmap can be exported as indices.
 *
 * What is stubbed: the TyrQuake engine symbols fisheye.c imports
 * (SURVEY.md section 8b "Imports"): console/cmd, zone, shell completion, the
 * software renderer entry points and the video globals.  `R_RenderView` paints
 * the caller-supplied synthetic globe face, `Draw_TileClear` paints the
 * caller-supplied background.
 *
 * Exports (all `ref_*`, plain C ABI, loaded with ctypes from tests/ and
 * bench.py's CPU-baseline leg only).
 */
#define _GNU_SOURCE
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "fisheye.c" /* the reference, in place (engine/NQ/fisheye.c) */

#include "engine_stubs.inc"

static int harness_displayed_plate(int k, int *platesize)
{
    int seen = 0;
    *platesize = globe.platesize;
    for (int i = 0; i < globe.numplates; i++) {
        if (globe.plates[i].display) {
            if (seen == k) return i;
            seen++;
        }
    }
    return -1;
}

/* ------------------------------------------------------------------------ */
/* exported harness API                                                      */
/* ------------------------------------------------------------------------ */
static byte *g_vidbuf;
static int g_inited;
static int g_alloc_w = -1, g_alloc_h = -1, g_alloc_ps = -1; /* sizes of lens/globe buffers */

/* basedir: directory containing lua-scripts/{globes,lenses}.  palette: 768 B RGB. */
int ref_init(const char *basedir, const unsigned char *palette768)
{
    if (g_inited) return -1;
    snprintf(com_basedir, sizeof com_basedir, "%s", basedir);
    memcpy(g_palette, palette768, 768);
    host_basepal = g_palette;
    g_ncmds = 0;
    F_Init();
    /* one-shot builds: never yield to the per-frame time slice (fisheye.c:819-826) */
    lens_builder.seconds_per_frame = 1.0e30f;
    g_inited = 1;
    return 0;
}

void ref_shutdown(void)
{
    if (!g_inited) return;
    F_Shutdown();
    g_inited = 0;
}

void ref_set_basedir(const char *basedir) { snprintf(com_basedir, sizeof com_basedir, "%s", basedir); }
void ref_set_write_dir(const char *dir) { snprintf(g_write_dir, sizeof g_write_dir, "%s", dir); }

void ref_command(const char *text) { Cmd_ExecuteString(text, src_command); }

const char *ref_log(void) { return g_log; }
void ref_log_clear(void) { g_log_len = 0; g_log[0] = 0; }
const char *ref_unhandled_commands(void) { return g_unhandled; }

/* Screen of w x h with the view rectangle (vx,vy,vw,vh) inside it and the given
 * row pitch, like vid/scr_vrect in the engine (include/vid.h:39-57). */
int ref_set_screen(int w, int h, int rowbytes, int vx, int vy, int vw, int vh)
{
    free(g_vidbuf);
    g_vidbuf = (byte *)calloc((size_t)rowbytes * h, 1);
    if (!g_vidbuf) return -1;
    vid.buffer = g_vidbuf;
    vid.width = w;
    vid.height = h;
    vid.rowbytes = rowbytes;
    vid.aspect = (float)w / (float)h;
    scr_vrect.x = vx;
    scr_vrect.y = vy;
    scr_vrect.width = vw;
    scr_vrect.height = vh;
    return 0;
}

/* One full engine frame through the real F_RenderView (platesize = min(w,h),
 * fisheye.c:707).  faces: [numplates][ps][ps]; background: [h][w]; out: [h][rowbytes]. */
int ref_frame(const unsigned char *faces, const unsigned char *background, unsigned char *out)
{
    g_faces = faces;
    g_background = background;
    g_render_calls = 0;
    /* F_RenderView only reallocates when the size differs from ITS previous call
     * (static pwidth/pheight, fisheye.c:700-727); if ref_build() resized the
     * buffers in between, put back buffers of the size F_RenderView assumes. */
    {
        int w = scr_vrect.width, h = scr_vrect.height, ps = w < h ? w : h;
        if (g_alloc_w != w || g_alloc_h != h || g_alloc_ps != ps) {
            free(globe.pixels);
            free(lens.pixels);
            free(lens.pixel_tints);
            globe.pixels = (byte *)malloc((size_t)ps * ps * MAX_PLATES);
            lens.pixels = (byte **)malloc((size_t)w * h * sizeof(byte *));
            lens.pixel_tints = (byte *)malloc((size_t)w * h);
            g_alloc_w = w; g_alloc_h = h; g_alloc_ps = ps;
            lens.changed = true;
        }
    }
    F_RenderView();
    while (lens_builder.working) resume_lensmap();
    if (out) memcpy(out, vid.buffer, (size_t)vid.rowbytes * vid.height);
    g_faces = NULL;
    g_background = NULL;
    return g_render_calls;
}

/* Lensmap (re)build with the plate size DECOUPLED from the screen size (the
 * BASELINE configs use 256/1024/2048-pixel faces).  This replays exactly the
 * rebuild branch of F_RenderView (fisheye.c:704-743) with `platesize` chosen by
 * the caller instead of min(w,h); every function called is the reference's. */
int ref_build(int width_px, int height_px, int platesize)
{
    lens.width_px = width_px;
    lens.height_px = height_px;
    globe.platesize = platesize;
    int area = width_px * height_px;

    if (globe.pixels) free(globe.pixels);
    if (lens.pixels) free(lens.pixels);
    if (lens.pixel_tints) free(lens.pixel_tints);
    globe.pixels = (byte *)malloc((size_t)platesize * platesize * MAX_PLATES);
    lens.pixels = (byte **)malloc((size_t)area * sizeof(byte *));
    lens.pixel_tints = (byte *)malloc((size_t)area);
    if (!globe.pixels || !lens.pixels || !lens.pixel_tints) return -1;
    g_alloc_w = width_px; g_alloc_h = height_px; g_alloc_ps = platesize;

    memset(lens.pixels, 0, (size_t)area * sizeof(byte *));
    memset(lens.pixel_tints, 255, (size_t)area);
    lens.valid = LUA_load_lens();
    if (!lens.valid) {
        strcpy(lens.name, "");
        Con_Printf("not a valid lens\n");
    }
    create_lensmap();
    while (lens_builder.working) resume_lensmap();
    lens.changed = globe.changed = zoom.changed = false;
    return (lens.valid && globe.valid) ? 0 : 1;
}

/* idx[i] = offset of the source texel inside globe.pixels, or -1 when unmapped */
void ref_get_lensmap(int *idx, unsigned char *tint)
{
    int area = lens.width_px * lens.height_px;
    for (int i = 0; i < area; i++) {
        idx[i] = lens.pixels[i] ? (int)(lens.pixels[i] - globe.pixels) : -1;
        if (tint) tint[i] = lens.pixel_tints[i];
    }
}

void ref_get_palmaps(unsigned char *out /* [6][256] */)
{
    for (int j = 0; j < MAX_PLATES; j++) memcpy(out + j * 256, globe.plates[j].palette, 256);
}

int ref_numplates(void) { return globe.numplates; }
int ref_platesize(void) { return globe.platesize; }
double ref_scale(void) { return lens.scale; }
int ref_map_type(void) { return (int)lens.map_type; }
int ref_lens_valid(void) { return lens.valid; }
int ref_globe_valid(void) { return globe.valid; }
int ref_rubix_enabled(void) { return rubix.enabled; }
double ref_lens_width(void) { return lens.width; }
double ref_lens_height(void) { return lens.height; }
int ref_max_fov(void) { return zoom.max_fov; }
int ref_max_vfov(void) { return zoom.max_vfov; }
int ref_fisheye_enabled(void) { return fisheye_enabled; }
double ref_plate_fov(void) { return fisheye_plate_fov; }

void ref_get_display(int *out /* [6] */)
{
    for (int i = 0; i < MAX_PLATES; i++) out[i] = i < globe.numplates ? globe.plates[i].display : 0;
}

/* out: per plate 11 floats: forward[3] right[3] up[3] fov dist */
void ref_get_plates(float *out)
{
    for (int i = 0; i < globe.numplates; i++) {
        float *o = out + i * 11;
        memcpy(o, globe.plates[i].forward, 12);
        memcpy(o + 3, globe.plates[i].right, 12);
        memcpy(o + 6, globe.plates[i].up, 12);
        o[9] = globe.plates[i].fov;
        o[10] = globe.plates[i].dist;
    }
}

/* The hot loop alone: render_lensmap() (fisheye.c:2406-2424) over caller faces.
 * faces: [6][ps][ps] (copied into globe.pixels), background/out: [vid.height][vid.rowbytes]. */
void ref_render(const unsigned char *faces, int numfaces, const unsigned char *background, unsigned char *out)
{
    size_t ps2 = (size_t)globe.platesize * globe.platesize;
    memcpy(globe.pixels, faces, ps2 * (size_t)numfaces);
    if (background) memcpy(vid.buffer, background, (size_t)vid.rowbytes * vid.height);
    render_lensmap();
    if (out) memcpy(out, vid.buffer, (size_t)vid.rowbytes * vid.height);
}

/* Times `reps` calls of render_lensmap() on the current lensmap/faces and
 * returns the best single-call wall time in seconds (CLOCK_MONOTONIC). */
double ref_time_render(int reps, double *total_seconds)
{
    double best = 1e30, total = 0;
    for (int r = 0; r < reps; r++) {
        struct timespec a, b;
        clock_gettime(CLOCK_MONOTONIC, &a);
        render_lensmap();
        clock_gettime(CLOCK_MONOTONIC, &b);
        double dt = (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
        if (dt < best) best = dt;
        total += dt;
    }
    if (total_seconds) *total_seconds = total;
    return best;
}

int ref_write_config(const char *path)
{
    FILE *f = fopen(path, "w");
    if (!f) return -1;
    F_WriteConfig(f);
    fclose(f);
    return 0;
}

/* direct probes of the reference's Lua<->C bridge, for interpreter parity tests */
int ref_lens_inverse(double x, double y, float *ray)
{
    vec3_t r = {0, 0, 0};
    if (lua_refs.lens_inverse == -1) return -2;
    int st = LUAtoC_lens_inverse(x, y, r);
    ray[0] = r[0]; ray[1] = r[1]; ray[2] = r[2];
    return st;
}

int ref_lens_forward(const float *ray, double *x, double *y)
{
    vec3_t r = {ray[0], ray[1], ray[2]};
    if (lua_refs.lens_forward == -1) return -2;
    return LUAtoC_lens_forward(r, x, y);
}

int ref_ray_to_plate(const float *ray, double *u, double *v)
{
    vec3_t r = {ray[0], ray[1], ray[2]};
    int p = ray_to_plate_index(r);
    if (p < 0) return -1;
    if (!ray_to_plate_uv(p, r, u, v)) return -2 - p;
    return p;
}
