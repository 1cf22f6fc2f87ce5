/* TEST INFRASTRUCTURE — parity oracle, not part of the product.  See blinky_oracle.h.
 *
 * Literal plain-C restatement of the reference's engine/NQ/fisheye.c for the
 * lens-warp path.  Float32/float64 truncation points are reproduced exactly:
 * `vec_t` is float (engine/include/mathlib.h:30), x86-64 evaluates float
 * expressions in float (FLT_EVAL_METHOD 0), and this file is compiled with
 * -ffp-contract=off and WITHOUT -ffast-math, like oracle/_ref.
 */
#include "blinky_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <pthread.h>
#include <unistd.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846 /* engine/include/mathlib.h:55 */
#endif

/* ------------------------------------------------------------------------ */
/* mathlib (engine/common/mathlib.c:349-429, engine/include/mathlib.h:70)    */
/* ------------------------------------------------------------------------ */
#define DOT(x, y) ((x)[0] * (y)[0] + (x)[1] * (y)[1] + (x)[2] * (y)[2]) /* float arithmetic on float operands */

static void vector_ma(const float a[3], const float scale, const float b[3], float c[3])
{ /* mathlib.c:349-355 */
    c[0] = a[0] + scale * b[0];
    c[1] = a[1] + scale * b[1];
    c[2] = a[2] + scale * b[2];
}

static void cross_product(const float v1[3], const float v2[3], float cross[3])
{ /* mathlib.c:388-394 */
    cross[0] = v1[1] * v2[2] - v1[2] * v2[1];
    cross[1] = v1[2] * v2[0] - v1[0] * v2[2];
    cross[2] = v1[0] * v2[1] - v1[1] * v2[0];
}

static float vector_normalize(float v[3])
{ /* mathlib.c:412-429: float length, double sqrt rounded back to float */
    float length, ilength;
    length = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    length = sqrt(length);
    if (length) {
        ilength = 1 / length;
        v[0] *= ilength;
        v[1] *= ilength;
        v[2] *= ilength;
    }
    return length;
}

/* ------------------------------------------------------------------------ */
/* globe loading (fisheye.c:1752-1875)                                       */
/* ------------------------------------------------------------------------ */
void orc_globe_set_plate(orc_globe *g, int i, const double forward[3], const double up[3], double fov_degrees)
{
    orc_plate *p = &g->plates[i];
    for (int j = 0; j < 3; j++) p->forward[j] = forward[j]; /* :1818 double -> float */
    for (int j = 0; j < 3; j++) p->up[j] = up[j];           /* :1843 */
    cross_product(p->up, p->forward, p->right);             /* :1849 */
    cross_product(p->forward, p->right, p->up);             /* :1850 (no normalisation) */
    p->fov = fov_degrees * M_PI / 180;                      /* :1858 double math, float store */
    p->dist = 0.5 / tan(p->fov / 2);                        /* :1868 */
    p->display = 0;
}

/* ------------------------------------------------------------------------ */
/* pure coordinate converters (fisheye.c:1184-1214)                          */
/* ------------------------------------------------------------------------ */
void orc_latlon_to_ray(double lat, double lon, float ray[3])
{ /* :1184-1190 */
    double clat = cos(lat);
    ray[0] = sin(lon) * clat;
    ray[1] = sin(lat);
    ray[2] = cos(lon) * clat;
}

void orc_ray_to_latlon(const float ray[3], double *lat, double *lon)
{ /* :1192-1196; ray[0]*ray[0]+ray[2]*ray[2] is a float expression */
    *lon = atan2(ray[0], ray[2]);
    *lat = atan2(ray[1], sqrt(ray[0] * ray[0] + ray[2] * ray[2]));
}

void orc_plate_uv_to_ray(const orc_globe *g, int plate, double u, double v, float ray[3])
{ /* :1198-1214 */
    u -= 0.5;
    v -= 0.5;
    v = -v;
    ray[0] = ray[1] = ray[2] = 0;
    vector_ma(ray, g->plates[plate].dist, g->plates[plate].forward, ray);
    vector_ma(ray, u, g->plates[plate].right, ray); /* double -> float at the call */
    vector_ma(ray, v, g->plates[plate].up, ray);
    vector_normalize(ray);
}

/* C->Lua wrappers: results pass through float32 vec3_t storage */
void orc_lua_latlon_to_ray(double lat, double lon, double out[3])
{ /* CtoLUA_latlon_to_ray :1494-1504 */
    float ray[3];
    orc_latlon_to_ray(lat, lon, ray);
    out[0] = ray[0];
    out[1] = ray[1];
    out[2] = ray[2];
}

void orc_lua_ray_to_latlon(double rx, double ry, double rz, double *lat, double *lon)
{ /* CtoLUA_ray_to_latlon :1506-1519: arguments narrowed to float first (:1512) */
    float ray[3] = {rx, ry, rz};
    orc_ray_to_latlon(ray, lat, lon);
}

int orc_lua_plate_to_ray(const orc_globe *g, double plate, double u, double v, double out[3])
{ /* CtoLUA_plate_to_ray :1521-1537: index truncated to int, nil when out of range */
    int plate_index = plate;
    float ray[3];
    if (plate_index < 0 || plate_index >= g->numplates) return 0;
    orc_plate_uv_to_ray(g, plate_index, u, v, ray);
    out[0] = ray[0];
    out[1] = ray[1];
    out[2] = ray[2];
    return 1;
}

/* ------------------------------------------------------------------------ */
/* zoom (fisheye.c:1293-1386)                                                */
/* ------------------------------------------------------------------------ */
int orc_calc_zoom(int zoom_type, int fov, int max_fov, int max_vfov, double lens_width, double lens_height,
                  int width_px, int height_px, orc_forward_fn fwd, void *ud, double *scale_out)
{
    double scale = -1; /* :1296 */

    if (zoom_type == ORC_ZOOM_FOV || zoom_type == ORC_ZOOM_VFOV) {
        if (max_fov <= 0 || max_vfov <= 0) return 0;                 /* :1301-1305 */
        else if (zoom_type == ORC_ZOOM_FOV && fov > max_fov) return 0;   /* :1306-1309 */
        else if (zoom_type == ORC_ZOOM_VFOV && fov > max_vfov) return 0; /* :1310-1313 */

        if (fwd) { /* :1316 */
            float ray[3];
            double x, y;
            double fovr = fov * M_PI / 180; /* :1319 */
            if (zoom_type == ORC_ZOOM_FOV) {
                orc_latlon_to_ray(0, fovr * 0.5, ray);                       /* :1321 */
                if (fwd(ray[0], ray[1], ray[2], &x, &y, ud) == 1)            /* :1322 (0 and -1 are both truthy-fail below) */
                    scale = x / (width_px * 0.5);                            /* :1323 */
                else
                    return 0;
            } else {
                orc_latlon_to_ray(fovr * 0.5, 0, ray);                       /* :1331 */
                if (fwd(ray[0], ray[1], ray[2], &x, &y, ud) == 1)
                    scale = y / (height_px * 0.5);                           /* :1333 */
                else
                    return 0;
            }
        } else {
            return 0; /* :1341-1345 */
        }
    } else if (zoom_type == ORC_ZOOM_CONTAIN || zoom_type == ORC_ZOOM_COVER) { /* :1347 */
        double fit_width_scale = lens_width / width_px;
        double fit_height_scale = lens_height / height_px;
        int width_provided = (lens_width > 0);
        int height_provided = (lens_height > 0);
        if (!width_provided && height_provided) {
            scale = fit_height_scale;
        } else if (width_provided && !height_provided) {
            scale = fit_width_scale;
        } else if (!width_provided && !height_provided) {
            return 0;
        } else {
            double lens_aspect = lens_width / lens_height;
            double screen_aspect = (double)width_px / height_px;
            int lens_wider = lens_aspect > screen_aspect;
            if (zoom_type == ORC_ZOOM_CONTAIN)
                scale = lens_wider ? fit_width_scale : fit_height_scale;
            else
                scale = lens_wider ? fit_height_scale : fit_width_scale;
        }
    }

    if (scale <= 0) return 0; /* :1380 (also catches ZOOM_NONE's -1) */
    *scale_out = scale;
    return 1;
}

/* NOTE on :1322 — `if (LUAtoC_lens_forward(...))` treats status -1 as true and
 * would use uninitialised x/y; no shipped lens returns -1 there, and this
 * restatement (like the product) fails the zoom instead. */

/* ------------------------------------------------------------------------ */
/* globe pixel getters (fisheye.c:2023-2066)                                 */
/* ------------------------------------------------------------------------ */
static int ray_to_plate_index(const orc_globe *g, const float ray[3])
{
    int plate_index = 0;
    if (g->plate_fn) { /* :2027-2033 */
        if (g->plate_fn(ray[0], ray[1], ray[2], &plate_index, g->plate_ud)) return plate_index;
        return -1;
    }
    double max_dp = -2; /* :2038 */
    for (int i = 0; i < g->numplates; ++i) {
        double dp = DOT(ray, g->plates[i].forward); /* float dot product widened */
        if (dp > max_dp) {
            max_dp = dp;
            plate_index = i;
        }
    }
    return plate_index;
}

static int ray_to_plate_uv(const orc_globe *g, int plate_index, const float ray[3], double *u, double *v)
{ /* :2052-2066 */
    const orc_plate *p = &g->plates[plate_index];
    double x = DOT(p->right, ray);
    double y = DOT(p->up, ray);
    double z = DOT(p->forward, ray);
    double dist = 0.5 / tan(p->fov / 2); /* float fov/2, double tan */
    *u = x / z * dist + 0.5;
    *v = -y / z * dist + 0.5;
    return *u >= 0 && *u <= 1 && *v >= 0 && *v <= 1;
}

/* ------------------------------------------------------------------------ */
/* lens pixel setters (fisheye.c:1922-2013)                                  */
/* ------------------------------------------------------------------------ */
typedef struct {
    orc_globe *g;
    const orc_rubix *rubix;
    orc_lensmap *lm;
} build_ctx;

static void set_lensmap_grid(build_ctx *c, int lx, int ly, int px, int py, int plate_index)
{ /* :1922-1960 */
    double block_size = (c->rubix->pad_size + c->rubix->cell_size);
    double num_units = c->rubix->numcells * block_size + c->rubix->pad_size;
    double unit_size_px = (double)c->g->platesize / num_units;
    double ux = (double)px / unit_size_px;
    double uy = (double)py / unit_size_px;
    int ongrid = fmod(ux, block_size) < c->rubix->pad_size || fmod(uy, block_size) < c->rubix->pad_size;
    if (!ongrid) c->lm->tint[lx + ly * c->lm->width_px] = plate_index;
}

static void set_lensmap_from_plate(build_ctx *c, int lx, int ly, int px, int py, int plate_index)
{ /* :1963-1982 */
    if (lx < 0 || lx >= c->lm->width_px || ly < 0 || ly >= c->lm->height_px) return;
    if (px < 0 || px >= c->g->platesize || py < 0 || py >= c->g->platesize) return;
    c->g->plates[plate_index].display = 1;
    /* GLOBEPIXEL(plate,x,y) - globe.pixels  (:349) */
    c->lm->idx[lx + ly * c->lm->width_px] = plate_index * c->g->platesize * c->g->platesize + px + py * c->g->platesize;
    set_lensmap_grid(c, lx, ly, px, py, plate_index);
}

static void set_lensmap_from_plate_uv(build_ctx *c, int lx, int ly, double u, double v, int plate_index)
{ /* :1985-1992 */
    int px = (int)(u * c->g->platesize);
    int py = (int)(v * c->g->platesize);
    set_lensmap_from_plate(c, lx, ly, px, py, plate_index);
}

static void set_lensmap_from_ray(build_ctx *c, int lx, int ly, double sx, double sy, double sz)
{ /* :1995-2013 */
    float ray[3] = {sx, sy, sz};
    int plate_index = ray_to_plate_index(c->g, ray);
    if (plate_index < 0) return;
    /* NB: a globe_plate() script may return an index >= numplates; the reference
     * then reads plates[] out of range (MAX_PLATES is not checked).  Shipped
     * globes never do; this oracle treats it as unmapped. */
    if (plate_index >= ORC_MAX_PLATES) return;
    double u, v;
    if (!ray_to_plate_uv(c->g, plate_index, ray, &u, &v)) return;
    set_lensmap_from_plate_uv(c, lx, ly, u, v, plate_index);
}

static void clear_lensmap(orc_globe *g, orc_lensmap *lm)
{
    int area = lm->width_px * lm->height_px;
    for (int i = 0; i < area; i++) lm->idx[i] = -1; /* memset(lens.pixels,0) :731 */
    memset(lm->tint, 255, (size_t)area);            /* :732 */
    for (int i = 0; i < g->numplates; i++) g->plates[i].display = 0; /* :2383-2385 */
}

/* ------------------------------------------------------------------------ */
/* inverse builder (fisheye.c:2084-2124 with 1545-1588)                      */
/* ------------------------------------------------------------------------ */
int orc_build_inverse(orc_globe *g, const orc_rubix *rubix, orc_lensmap *lm, orc_inverse_fn inv, void *ud)
{
    build_ctx c = {g, rubix, lm};
    clear_lensmap(g, lm);
    for (int ly = lm->height_px - 1; ly >= 0; --ly) {               /* :2093, :2349 */
        double y = -(ly - lm->height_px / 2) * lm->scale;           /* :2100 (integer /2) */
        for (int lx = 0; lx < lm->width_px; ++lx) {
            double x = (lx - lm->width_px / 2) * lm->scale;         /* :2105 */
            double r[3];
            int status = inv(x, y, r, ud);                          /* :2109 */
            if (status == 0) continue;
            else if (status == -1) return -1;
            /* LUAtoC_lens_inverse :1559-1562: float store + VectorNormalize */
            float ray[3] = {r[0], r[1], r[2]};
            vector_normalize(ray);
            set_lensmap_from_ray(&c, lx, ly, ray[0], ray[1], ray[2]); /* :2118 */
        }
    }
    return 0;
}

/* ------------------------------------------------------------------------ */
/* forward builder (fisheye.c:2126-2338)                                     */
/* ------------------------------------------------------------------------ */
typedef struct {
    build_ctx *c;
    orc_forward_fn fwd;
    void *ud;
} fwd_ctx;

static int uv_to_screen(fwd_ctx *f, int plate_index, double u, double v, int *lx, int *ly)
{ /* :2227-2243 */
    float ray[3];
    orc_plate_uv_to_ray(f->c->g, plate_index, u, v, ray);
    double x, y;
    int status = f->fwd(ray[0], ray[1], ray[2], &x, &y, f->ud);
    if (status == 0 || status == -1) return status;
    *lx = (int)(x / f->c->lm->scale + f->c->lm->width_px / 2);
    *ly = (int)(-y / f->c->lm->scale + f->c->lm->height_px / 2);
    return status;
}

static void draw_quad(build_ctx *c, int *tl, int *tr, int *bl, int *br, int plate_index, int px, int py)
{ /* :2246-2338 */
    int *p[] = {tl, tr, br, bl};
    int x = tl[0], y = tl[1];
    int miny = y, maxy = y;
    int minx = x, maxx = x;
    int i;
    for (i = 1; i < 4; i++) {
        int tx = p[i][0];
        if (tx < minx) { minx = tx; }
        else if (tx > maxx) { maxx = tx; }
        int ty = p[i][1];
        if (ty < miny) { miny = ty; }
        else if (ty > maxy) { maxy = ty; }
    }
    const int maxdiff = 20;
    if (abs(minx - maxx) > maxdiff || abs(miny - maxy) > maxdiff) return;

    if (miny == maxy && minx == maxx) {
        set_lensmap_from_plate(c, x, y, px, py, plate_index);
        return;
    }
    if (miny == maxy) {
        for (int tx = minx; tx <= maxx; ++tx) set_lensmap_from_plate(c, tx, miny, px, py, plate_index);
        return;
    }
    if (minx == maxx) {
        for (int ty = miny; ty <= maxy; ++ty) set_lensmap_from_plate(c, x, ty, px, py, plate_index);
        return;
    }
    for (y = miny; y <= maxy; ++y) {
        int tx[2] = {minx, maxx};
        int txi = 0;
        int j = 3;
        for (i = 0; i < 4; ++i) {
            int ix = p[i][0], iy = p[i][1];
            int jx = p[j][0], jy = p[j][1];
            if ((iy < y && y <= jy) || (jy < y && y <= iy)) {
                double dy = jy - iy;
                double dx = jx - ix;
                tx[txi] = (int)(ix + (y - iy) / dy * dx);
                if (++txi == 2) break;
            }
            j = i;
        }
        if (tx[0] > tx[1]) {
            int temp = tx[0];
            tx[0] = tx[1];
            tx[1] = temp;
        }
        if (tx[1] - tx[0] > maxdiff) return; /* :2327-2331 (prints and aborts the quad) */
        for (x = tx[0]; x <= tx[1]; ++x) set_lensmap_from_plate(c, x, y, px, py, plate_index);
    }
}

int orc_build_forward(orc_globe *g, const orc_rubix *rubix, orc_lensmap *lm, orc_forward_fn fwd, void *ud)
{
    build_ctx c = {g, rubix, lm};
    fwd_ctx f = {&c, fwd, ud};
    clear_lensmap(g, lm);
    int platesize = g->platesize;
    /* :2357-2358 malloc()s these without initialising them; when lens_forward
     * returns nil for a corner the stale entry is used (:2155 `continue`).  The
     * reference's result is then undefined; zero-filled here. */
    int *rowa = calloc((size_t)(platesize + 1), sizeof(int[2]));
    int *rowb = calloc((size_t)(platesize + 1), sizeof(int[2]));
    int *top = rowa, *bot = rowb;
    int rc = 0;

    for (int plate_index = 0; plate_index < g->numplates && rc == 0; ++plate_index) { /* :2135 */
        int px;
        for (int py = platesize - 1; py >= 0 && rc == 0; --py) {                      /* :2138, :2361, :2209 */
            if (py == platesize - 1) {                                                 /* :2148 lower points */
                double v = (py + 0.5) / platesize;
                for (px = 0; px < platesize; ++px) {
                    if (px == 0) {
                        double u = (px - 0.5) / platesize;
                        int status = uv_to_screen(&f, plate_index, u, v, &bot[0], &bot[1]);
                        if (status == 0) continue; else if (status == -1) { rc = -1; break; }
                    }
                    double u = (px + 0.5) / platesize;
                    int index = 2 * (px + 1);
                    int status = uv_to_screen(&f, plate_index, u, v, &bot[index], &bot[index + 1]);
                    if (status == 0) continue; else if (status == -1) { rc = -1; break; }
                }
                if (rc) break;
            } else { /* :2164-2169 */
                int *temp = top;
                top = bot;
                bot = temp;
            }
            double v = (py - 0.5) / platesize; /* :2172 upper points */
            for (px = 0; px < platesize; ++px) {
                if (px == 0) {
                    double u = (px - 0.5) / platesize;
                    int status = uv_to_screen(&f, plate_index, u, v, &top[0], &top[1]);
                    if (status == 0) continue; else if (status == -1) { rc = -1; break; }
                }
                double u = (px + 0.5) / platesize;
                int index = 2 * (px + 1);
                int status = uv_to_screen(&f, plate_index, u, v, &top[index], &top[index + 1]);
                if (status == 0) continue; else if (status == -1) { rc = -1; break; }
            }
            if (rc) break;

            v = ((double)py) / platesize; /* :2189 */
            for (px = 0; px < platesize; ++px) {
                double u = ((double)px) / platesize;
                float ray[3];
                orc_plate_uv_to_ray(g, plate_index, u, v, ray);
                if (plate_index != ray_to_plate_index(g, ray)) continue; /* :2196 */
                int index = 2 * px;
                draw_quad(&c, &top[index], &top[index + 2], &bot[index], &bot[index + 2], plate_index, px, py);
            }
        }
    }
    free(rowa);
    free(rowb);
    return rc;
}

/* ------------------------------------------------------------------------ */
/* palette (fisheye.c:835-908)                                               */
/* ------------------------------------------------------------------------ */
static int find_closest_pal_index(const uint8_t *basepal, int r, int g, int b)
{ /* :835-855 */
    int mindist = 256 * 256 * 256;
    int minindex = 0;
    const uint8_t *pal = basepal;
    for (int i = 0; i < 256; ++i) {
        int dr = (int)pal[0] - r;
        int dg = (int)pal[1] - g;
        int db = (int)pal[2] - b;
        int dist = dr * dr + dg * dg + db * db;
        if (dist < mindist) {
            mindist = dist;
            minindex = i;
        }
        pal += 3;
    }
    return minindex;
}

void orc_create_palmap(const uint8_t palette[768], uint8_t out[ORC_MAX_PLATES][256])
{ /* :857-908 */
    int percent = 256 / 6;
    int tint[3];
    for (int j = 0; j < ORC_MAX_PLATES; ++j) {
        tint[0] = tint[1] = tint[2] = 0;
        switch (j) {
            case 0: tint[0] = tint[1] = tint[2] = 255; break;
            case 1: tint[2] = 255; break;
            case 2: tint[0] = 255; break;
            case 3: tint[0] = tint[1] = 255; break;
            case 4: tint[0] = tint[2] = 255; break;
            case 5: tint[1] = tint[2] = 255; break;
        }
        const uint8_t *pal = palette;
        for (int i = 0; i < 256; ++i) {
            int r = pal[0];
            int g = pal[1];
            int b = pal[2];
            r += percent * (tint[0] - r) >> 8; /* `+=` binds looser than `>>`: r += ((percent*(t-r)) >> 8) */
            g += percent * (tint[1] - g) >> 8;
            b += percent * (tint[2] - b) >> 8;
            if (r < 0) r = 0;
            if (r > 255) r = 255;
            if (g < 0) g = 0;
            if (g > 255) g = 255;
            if (b < 0) b = 0;
            if (b > 255) b = 255;
            out[j][i] = find_closest_pal_index(palette, r, g, b);
            pal += 3;
        }
    }
}

/* ------------------------------------------------------------------------ */
/* THE hot loop: render_lensmap (fisheye.c:2406-2424)                        */
/* ------------------------------------------------------------------------ */
static void render_rows(const orc_lensmap *lm, const uint8_t *faces, const uint8_t palmaps[ORC_MAX_PLATES][256],
                        int rubix_enabled, uint8_t *vbuf, int rowbytes, int vrect_x, int vrect_y, int y0, int y1)
{
    const int32_t *lmap = lm->idx + (size_t)y0 * lm->width_px;
    const uint8_t *pmap = lm->tint + (size_t)y0 * lm->width_px;
    for (int y = y0; y < y1; y++)
        for (int x = 0; x < lm->width_px; x++, lmap++, pmap++)
            if (*lmap >= 0) { /* `if (*lmap)` — non-NULL pointer */
                int lx = x + vrect_x;
                int ly = y + vrect_y;
                uint8_t src = faces[*lmap];
                if (rubix_enabled) {
                    int i = *pmap;
                    vbuf[lx + (size_t)ly * rowbytes] = i != 255 ? palmaps[i][src] : src;
                } else {
                    vbuf[lx + (size_t)ly * rowbytes] = src;
                }
            }
}

void orc_render_lensmap(const orc_lensmap *lm, const uint8_t *faces, const uint8_t palmaps[ORC_MAX_PLATES][256],
                        int rubix_enabled, uint8_t *vbuf, int rowbytes, int vrect_x, int vrect_y)
{
    render_rows(lm, faces, palmaps, rubix_enabled, vbuf, rowbytes, vrect_x, vrect_y, 0, lm->height_px);
}

typedef struct {
    const orc_lensmap *lm;
    const uint8_t *faces;
    const uint8_t (*palmaps)[256];
    int rubix_enabled;
    uint8_t *vbuf;
    int rowbytes, vrect_x, vrect_y, y0, y1;
} row_job;

static void *row_worker(void *arg)
{
    row_job *j = (row_job *)arg;
    render_rows(j->lm, j->faces, j->palmaps, j->rubix_enabled, j->vbuf, j->rowbytes, j->vrect_x, j->vrect_y, j->y0, j->y1);
    return NULL;
}

/* Row bands on `threads` POSIX threads (the reference itself is single
 * threaded; this is the "all host cores" CPU baseline).  Name kept from the
 * OpenMP plan in BASELINE.md; pthreads are used because the image's default
 * compiler wrapper ships no libgomp. */
void orc_render_lensmap_omp(const orc_lensmap *lm, const uint8_t *faces, const uint8_t palmaps[ORC_MAX_PLATES][256],
                            int rubix_enabled, uint8_t *vbuf, int rowbytes, int vrect_x, int vrect_y, int threads)
{
    if (threads < 1) threads = orc_max_threads();
    if (threads > 256) threads = 256;
    pthread_t tid[256];
    row_job jobs[256];
    for (int t = 0; t < threads; t++) {
        row_job j = {lm, faces, palmaps, rubix_enabled, vbuf, rowbytes, vrect_x, vrect_y,
                     (int)((long)lm->height_px * t / threads), (int)((long)lm->height_px * (t + 1) / threads)};
        jobs[t] = j;
        if (pthread_create(&tid[t], NULL, row_worker, &jobs[t]) != 0) {
            row_worker(&jobs[t]);
            tid[t] = 0;
        }
    }
    for (int t = 0; t < threads; t++)
        if (tid[t]) pthread_join(tid[t], NULL);
}

int orc_max_threads(void)
{
    long n = sysconf(_SC_NPROCESSORS_ONLN);
    return n > 0 ? (int)n : 1;
}

/* Wall-clock timing of the restated hot loop for the CPU baseline: `reps` calls,
 * returns the best single call in seconds, *total_seconds the sum. */
#include <time.h>
double orc_time_render(const orc_lensmap *lm, const uint8_t *faces, const uint8_t palmaps[ORC_MAX_PLATES][256],
                       int rubix_enabled, uint8_t *vbuf, int rowbytes, int threads, int reps, double *total_seconds)
{
    double best = 1e30, total = 0;
    for (int r = 0; r < reps; r++) {
        struct timespec a, b;
        clock_gettime(CLOCK_MONOTONIC, &a);
        if (threads > 1) orc_render_lensmap_omp(lm, faces, palmaps, rubix_enabled, vbuf, rowbytes, 0, 0, threads);
        else orc_render_lensmap(lm, faces, palmaps, rubix_enabled, vbuf, rowbytes, 0, 0);
        clock_gettime(CLOCK_MONOTONIC, &b);
        double dt = (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
        if (dt < best) best = dt;
        total += dt;
    }
    if (total_seconds) *total_seconds = total;
    return best;
}
