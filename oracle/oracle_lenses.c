/* TEST INFRASTRUCTURE — parity oracle, not part of the product.  See blinky_oracle.h.
 *
 * Literal C transcriptions of shipped Blinky lens and globe scripts
 * (the reference's game/lua-scripts/{lenses,globes}/<name>.lua).  A Lua 5.2 VM
 * executes those scripts as IEEE-double operations in source order with
 * libm for math.*; these functions perform the same operations in the same
 * order, so a correct Lua evaluator must reproduce their results BIT FOR BIT.
 * That is how the product's own Lua-subset evaluator (no real Lua exists in the
 * build image) is pinned independently of itself.
 *
 * Compiled with -ffp-contract=off and no -ffast-math.  `pi` is math.pi.
 */
#include <math.h>
#include <string.h>

#include "blinky_oracle.h"

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
static const double pi = M_PI;

/* ---- lenses/panini.lua ---------------------------------------------------- */
static const double panini_d = 1; /* :1 */

static int panini_inverse(double x, double y, double r[3], void *ud)
{ /* :8-17 */
    (void)ud;
    double d = panini_d;
    double k = x * x / ((d + 1) * (d + 1));
    double dscr = k * k * d * d - (k + 1) * (k * d * d - 1);
    double clon = (-k * d + sqrt(dscr)) / (k + 1);
    double S = (d + 1) / (d + clon);
    double lon = atan2(x, S * clon);
    double lat = atan2(y, S);
    orc_lua_latlon_to_ray(lat, lon, r);
    return 1;
}

static int panini_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :19-25 */
    (void)ud;
    double d = panini_d, lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    double S = (d + 1) / (d + cos(lon));
    *ox = S * sin(lon);
    *oy = S * tan(lat);
    return 1;
}

/* ---- lenses/stereographic.lua --------------------------------------------- */
static const double stereo_angleScale = 0.5; /* :1 */

static int stereographic_inverse(double x, double y, double o[3], void *ud)
{ /* :8-14 — r == 0 at the centre pixel gives NaN, by design of the script */
    (void)ud;
    double r = sqrt(x * x + y * y);
    double theta = atan(r) / stereo_angleScale;
    double s = sin(theta);
    o[0] = x / r * s;
    o[1] = y / r * s;
    o[2] = cos(theta);
    return 1;
}

static int stereographic_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :16-23 */
    (void)ud;
    double theta = acos(z);
    double r = tan(theta * stereo_angleScale);
    double c = r / sqrt(x * x + y * y);
    *ox = x * c;
    *oy = y * c;
    return 1;
}

/* ---- lenses/rectilinear.lua ----------------------------------------------- */
static int rectilinear_inverse(double x, double y, double o[3], void *ud)
{ /* :7-14 */
    (void)ud;
    double r = sqrt(x * x + y * y);
    double theta = atan(r);
    double s = sin(theta);
    o[0] = x / r * s;
    o[1] = y / r * s;
    o[2] = cos(theta);
    return 1;
}

static int rectilinear_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :16-23 */
    (void)ud;
    double theta = acos(z);
    double r = tan(theta);
    double c = r / sqrt(x * x + y * y);
    *ox = x * c;
    *oy = y * c;
    return 1;
}

/* ---- lenses/equirect.lua --------------------------------------------------- */
static int equirect_inverse(double x, double y, double o[3], void *ud)
{ /* :9-16 */
    (void)ud;
    if (fabs(y) > pi / 2 || fabs(x) > pi) return 0;
    double lon = x;
    double lat = y;
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int equirect_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :18-23 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon;
    *oy = lat;
    return 1;
}

/* ---- lenses/cylinder.lua --------------------------------------------------- */
static int cylinder_inverse(double x, double y, double o[3], void *ud)
{ /* :8-15 */
    (void)ud;
    if (fabs(x) > pi) return 0;
    double lon = x;
    double lat = atan(y);
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int cylinder_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :17-22 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon;
    *oy = tan(lat);
    return 1;
}

/* ---- lenses/mercator.lua --------------------------------------------------- */
static int mercator_inverse(double x, double y, double o[3], void *ud)
{ /* :12-19 */
    (void)ud;
    if (fabs(x) > pi) return 0;
    double lon = x;
    double lat = atan(sinh(y));
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int mercator_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :22-27 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon;
    *oy = log(tan(pi * 0.25 + lat * 0.5));
    return 1;
}

/* ---- lenses/hammer.lua ----------------------------------------------------- */
static int hammer_inverse(double x, double y, double o[3], void *ud)
{ /* :9-17 */
    (void)ud;
    if (x * x / 8 + y * y / 2 > 1) return 0;
    double z = sqrt(1 - 0.0625 * x * x - 0.25 * y * y);
    double lon = 2 * atan(z * x / (2 * (2 * z * z - 1)));
    double lat = asin(z * y);
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int hammer_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :19-24 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = 2 * sqrt(2) * cos(lat) * sin(lon * 0.5) / sqrt(1 + cos(lat) * cos(lon * 0.5));
    *oy = sqrt(2) * sin(lat) / sqrt(1 + cos(lat) * cos(lon * 0.5));
    return 1;
}

/* ---- lenses/fisheye1.lua --------------------------------------------------- */
static int fisheye1_inverse(double x, double y, double o[3], void *ud)
{ /* :9-20 */
    (void)ud;
    double r = sqrt(x * x + y * y);
    if (r > pi) return 0;
    double theta = r;
    double s = sin(theta);
    o[0] = x / r * s;
    o[1] = y / r * s;
    o[2] = cos(theta);
    return 1;
}

static int fisheye1_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :22-29 */
    (void)ud;
    double theta = acos(z);
    double r = theta;
    double c = r / sqrt(x * x + y * y);
    *ox = x * c;
    *oy = y * c;
    return 1;
}

/* ---- lenses/fisheye2.lua --------------------------------------------------- */
static int fisheye2_inverse(double x, double y, double o[3], void *ud)
{ /* :11-23 */
    (void)ud;
    double maxr = 2 * sin(pi * 0.5); /* :1 */
    double r = sqrt(x * x + y * y);
    if (r > maxr) return 0;
    double theta = 2 * asin(r * 0.5);
    double s = sin(theta);
    o[0] = x / r * s;
    o[1] = y / r * s;
    o[2] = cos(theta);
    return 1;
}

static int fisheye2_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :25-32 */
    (void)ud;
    double theta = acos(z);
    double r = 2 * sin(theta * 0.5);
    double c = r / sqrt(x * x + y * y);
    *ox = x * c;
    *oy = y * c;
    return 1;
}

/* ---- lenses/sinusoidal.lua, winkel1.lua (forward-only) ---------------------- */
static int sinusoidal_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* sinusoidal.lua:10-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon * cos(lat);
    *oy = lat;
    return 1;
}

static int winkel1_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* winkel1.lua:10-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon * (2 / pi + cos(lat)) / 2;
    *oy = lat;
    return 1;
}

/* ---- lenses/quincuncial.lua ------------------------------------------------ */
static const double q_eps = 0.0001;        /* :1 */
#define q_halfpi (pi / 2)                  /* :2 */

static double q_asqrt(double x)
{ /* :9-14 */
    if (x > 0) return sqrt(x);
    return 0;
}

/* :15-62; returns sn, cn, dn (the 4th result, ph, is unused by callers) */
static void q_ellipj(double u, double m, double *sn, double *cn, double *dn)
{
    double ai, b, phi, t, twon;
    if (m < q_eps) { /* :17-25 */
        t = sin(u);
        b = cos(u);
        ai = .25 * m * (u - t * b);
        *sn = t - ai * b;
        *cn = b + ai * t;
        *dn = 1 - .5 * m * t * t;
        return;
    }
    if (m >= 1 - q_eps) { /* :26-36 */
        ai = .25 * (1 - m);
        b = cosh(u);
        t = tanh(u);
        phi = 1 / b;
        twon = b * sinh(u);
        *sn = t + ai * (twon - u) / (b * b);
        *cn = phi - ai * t * phi * (twon - u);
        *dn = phi + ai * t * phi * (twon + u);
        return;
    }
    double a[10] = {0, 1, 0, 0, 0, 0, 0, 0, 0, 0}; /* 1-based like the Lua tables (:38-39) */
    double c[10] = {0, sqrt(m), 0, 0, 0, 0, 0, 0, 0, 0};
    int i = 1;
    b = sqrt(1 - m);
    twon = 1;
    while (fabs(c[i] / a[i]) > q_eps && i < 9) { /* :44-51 */
        ai = a[i];
        i = i + 1;
        c[i] = .5 * (ai - b);
        a[i] = .5 * (ai + b);
        b = q_asqrt(ai * b);
        twon = twon * 2;
    }
    phi = twon * a[i] * u; /* :53 */
    do {                   /* :54-59 */
        b = phi;
        t = c[i] * sin(b) / a[i];
        phi = .5 * (asin(t) + phi);
        i = i - 1;
    } while (!(i == 1));
    t = cos(phi);
    *sn = sin(phi);
    *cn = t;
    *dn = t / cos(phi - b);
}

static void q_cnrectify(double x, double y, double *latp, double *longd)
{ /* :74-104 */
    double sqrt2 = sqrt(2);       /* :69 */
    double sqrt22 = sqrt2 / 2;    /* :70 */
    double m = 1.0 / 2;           /* :71 */
    double ke = 1.85407467730137; /* :72 */
    double xpr = ke * (sqrt22 * x - sqrt22 * y) / sqrt2 + ke;
    double ypr = ke * (sqrt22 * x + sqrt22 * y) / sqrt2;
    double x1, y1;
    if (fabs(ypr) < q_eps) {
        double sni, cni, dni;
        q_ellipj(xpr, m, &sni, &cni, &dni);
        x1 = cni;
        y1 = 0.0;
    } else {
        double phi = xpr, psi = ypr;
        double s, c, d, s1, c1, d1;
        q_ellipj(phi, m, &s, &c, &d);
        q_ellipj(psi, 1 - m, &s1, &c1, &d1);
        double delta = pow(c1, 2) + m * pow(s, 2) * pow(s1, 2);
        x1 = (c * c1) / delta;
        y1 = -(s * d * s1 * d1) / delta;
    }
    *longd = atan2(y1, x1);
    *latp = 2 * atan2(sqrt(x1 * x1 + y1 * y1), 1) - q_halfpi;
}

static void q_rotate(double a, double b, double angle, double *a0, double *b0)
{ /* :153-159 */
    double c = cos(angle);
    double s = sin(angle);
    *a0 = a * c - b * s;
    *b0 = a * s + b * c;
}

static int q_inverse_intermediate(double x, double y, double o[3])
{ /* :161-172 */
    if (fabs(x) > 2 || fabs(y) > 1) return 0;
    x = x + 1;
    double lat, lon, r[3];
    q_cnrectify(x, y, &lat, &lon);
    orc_lua_latlon_to_ray(lat, -lon, r);
    o[0] = r[0];
    o[1] = r[2];
    o[2] = -r[1];
    return 1;
}

static int quincuncial_inverse(double x, double y, double o[3], void *ud)
{ /* :174-210 */
    (void)ud;
    double sqrt2 = sqrt(2);
    if (fabs(x) > sqrt2 || fabs(y) > sqrt2) return 0;
    double x0, y0;
    if (fabs(x) + fabs(y) < sqrt2) {
        q_rotate(x, y, pi / 4, &x0, &y0);
        x0 = x0 - 1;
    } else if (x > 0 && y < 0) {
        q_rotate(x, y, pi / 4, &x0, &y0);
        x0 = x0 - 1;
    } else if (x < 0 && y > 0) {
        q_rotate(x, y, pi / 4, &x0, &y0);
        x0 = x0 + 3;
    } else if (x < 0 && y < 0) {
        q_rotate(x, y, pi / 4 + pi, &x0, &y0);
        x0 = x0 + 1;
        y0 = y0 - 2;
    } else {
        q_rotate(x, y, pi / 4 + pi, &x0, &y0);
        x0 = x0 + 1;
        y0 = y0 + 2;
    }
    return q_inverse_intermediate(x0, y0, o);
}


/* ---- lenses/mollweide.lua --------------------------------------------------- */
static double mollweide_solveTheta(double lat)
{ /* :11-19 — Newton iteration, `repeat ... until dt < 0.001` (signed test, as written) */
    double t = lat, dt;
    do {
        dt = -(t + sin(t) - pi * sin(lat)) / (1 + cos(t));
        t = t + dt;
    } while (!(dt < 0.001));
    return t / 2;
}

static int mollweide_inverse(double x, double y, double o[3], void *ud)
{ /* :21-29 */
    (void)ud;
    const double root2 = sqrt(2); /* :1 */
    if (x * x / 8 + y * y / 2 > 1) return 0;
    double t = asin(y / root2);
    double lon = pi * x / (2 * root2 * cos(t));
    double lat = asin((2 * t + sin(2 * t)) / pi);
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int mollweide_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :31-37 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    double t = mollweide_solveTheta(lat);
    *ox = 2 * sqrt(2) / pi * lon * cos(t);
    *oy = sqrt(2) * sin(t);
    return 1;
}

/* ---- lenses/vandergrinten.lua ---------------------------------------------- */
static int vandergrinten_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :6-35 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    if (lat == 0) {
        *ox = lon;
        *oy = 0;
        return 1;
    }
    double t = asin(fabs(2 * lat / pi));
    if (fabs(lat) == pi / 2) {
        double y2 = pi * tan(t / 2);
        if (y2 * lat < 0) y2 = -y2;
        *ox = 0;
        *oy = y2;
        return 1;
    }
    double a = 0.5 * fabs(pi / lon - lon / pi);
    double g = cos(t) / (sin(t) + cos(t) - 1);
    double p = g * (2 / sin(t) - 1);
    double q = a * a + g;
    double xx = pi * (a * (g - p * p) + sqrt(a * a * (g - p * p) * (g - p * p) - (p * p + a * a) * (g * g - p * p))) / (p * p + a * a);
    double yy = pi * (p * q - a * sqrt((a * a + 1) * (p * p + a * a) - q * q)) / (p * p + a * a);
    if (lon * xx < 0) xx = -xx;
    if (lat * yy < 0) yy = -yy;
    *ox = xx;
    *oy = yy;
    return 1;
}

static double vandergrinten_maxr(void)
{ /* :109 — maxr = lens_forward(latlon_to_ray(0,pi)): the first of the two results */
    double r[3], mx, my;
    orc_lua_latlon_to_ray(0, pi, r);
    vandergrinten_forward(r[0], r[1], r[2], &mx, &my, NULL);
    return mx;
}

static int vandergrinten_inverse(double x, double y, double o[3], void *ud)
{ /* :46-107 (constants :37-44) */
    (void)ud;
    const double TOL = 1.e-10, THIRD = .33333333333333333333, C2_27 = .07407407407407407407, PI4_3 = 4.18879020478639098458,
                 PISQ = 9.86960440108935861869, TPISQ = 19.73920880217871723738, HPISQ = 4.93480220054467930934;
    const double maxr = vandergrinten_maxr();
    if (x * x + y * y > maxr * maxr) return 0;
    double lat, lon;
    double t, c0, c1, c2, c3, al, r2, r, m, d, ay, x2, y2;
    x2 = x * x;
    ay = fabs(y);
    if (ay < TOL) {
        lat = 0;
        t = x2 * x2 + TPISQ * (x2 + HPISQ);
        if (fabs(x) <= TOL) lon = 0;
        else lon = 0.5 * (x2 - PISQ + sqrt(t)) / x;
        orc_lua_latlon_to_ray(lat, lon, o);
        return 1;
    }
    y2 = y * y;
    r = x2 + y2;
    r2 = r * r;
    c1 = -pi * ay * (r + PISQ);
    c3 = r2 + (2 * pi) * (ay * r + pi * (y2 + pi * (ay + pi / 2)));
    c2 = c1 + PISQ * (r - 3 * y2);
    c0 = pi * ay;
    c2 = c2 / c3;
    al = c1 / c3 - THIRD * c2 * c2;
    m = 2 * sqrt(-THIRD * al);
    d = C2_27 * c2 * c2 * c2 + (c0 * c0 - THIRD * c2 * c1) / c3;
    d = 3 * d / (al * m);
    t = fabs(d);
    if (t - TOL <= 1) {
        if (t > 1) {
            if (d > 0) d = 0;
            else d = pi;
        } else {
            d = acos(d);
        }
        lat = pi * (m * cos(d * THIRD + PI4_3) - THIRD * c2);
        if (y < 0) lat = -lat;
        t = r2 + TPISQ * (x2 - y2 + HPISQ);
        if (fabs(x) <= TOL) {
            lon = 0;
        } else {
            if (t <= 0) lon = 0.5 * (r - PISQ) / x;
            else lon = 0.5 * (r - PISQ + sqrt(t)) / x;
        }
    } else {
        return 0;
    }
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

/* ---- lenses/cube.lua -------------------------------------------------------- */
static void cube_modf_cell(double n, double *i, double *f)
{ /* col()/row() :12-28: math.modf, cells left of / above zero shifted down by one */
    double ip;
    double fp = modf(n, &ip);
    if (n < 0) {
        *i = ip - 1;
        *f = fp + 1;
    } else {
        *i = ip;
        *f = fp;
    }
}

static int cube_inverse(double x, double y, double o[3], void *ud)
{ /* :30-71 */
    (void)ud;
    const double cols = 4, rows = 3;
    double r, v, c, u;
    x = x - 0.5;
    cube_modf_cell(-y + rows / 2, &r, &v);
    cube_modf_cell(x + cols / 2, &c, &u);
    u = u - 0.5;
    v = v - 0.5;
    v = -v;
    if (r < 0 || r >= rows || c < -1 || c >= cols) return 0;
    if (r == 0 || r == 2) {
        if (!(c == 1)) return 0;
    }
    if (r == 0) { o[0] = u; o[1] = 0.5; o[2] = -v; }          /* top */
    else if (r == 2) { o[0] = u; o[1] = -0.5; o[2] = v; }     /* bottom */
    else if (c == 0) { o[0] = -0.5; o[1] = v; o[2] = u; }     /* left */
    else if (c == 1) { o[0] = u; o[1] = v; o[2] = 0.5; }      /* front */
    else if (c == 2) { o[0] = 0.5; o[1] = v; o[2] = -u; }     /* right */
    else if (c == 3 || c == -1) { o[0] = -u; o[1] = v; o[2] = -0.5; } /* back */
    else return 0;
    return 1;
}

static int cube_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :73-125 — "only to be used for FOV" */
    (void)ud;
    double ax = fabs(x), ay = fabs(y), az = fabs(z);
    double mx = ax > ay ? ax : ay; /* math.max(ax,ay,az) */
    mx = mx > az ? mx : az;
    double u, v;
    if (mx == ax) {
        if (x > 0) { u = -z / x * 0.5; v = y / x * 0.5; *ox = 1 + u; *oy = v; }
        else { u = z / -x * 0.5; v = y / -x * 0.5; *ox = -1 + u; *oy = v; }
        return 1;
    } else if (mx == ay) {
        if (y > 0) { u = x / y * 0.5; v = -z / y * 0.5; *ox = u; *oy = 1 + v; }
        else { u = x / -y * 0.5; v = z / -y * 0.5; *ox = u; *oy = -1 + v; }
        return 1;
    } else if (mx == az) {
        if (z > 0) { u = x / z * 0.5; v = y / z * 0.5; *ox = u; *oy = v; }
        else {
            u = -x / -z * 0.5;
            v = y / -z * 0.5;
            if (u > 0) *ox = -2 + u;
            else *ox = 2 + u;
            *oy = v;
        }
        return 1;
    }
    return -1; /* the script falls off its end: no values */
}

/* ---- registry --------------------------------------------------------------- */
/* ---- lenses/winkeltripel.lua ---------------------------------------------- */
static double wt_lens_width, wt_lens_height, wt_artifact_x, wt_artifact_y; /* :82-94, set by wt_onload() */

static int winkeltripel_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :9-21 */
    (void)ud;
    const double clat0 = 2 / pi; /* :2 */
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    double clat = cos(lat);
    double temp = clat * cos(lon * 0.5);
    double D = acos(temp);
    double C = 1 - temp * temp;
    temp = D / sqrt(C);
    *ox = 0.5 * (2 * temp * clat * sin(lon * 0.5) + lon * clat0);
    *oy = 0.5 * (temp * sin(lat) + lat);
    return 1;
}

static int winkeltripel_inverse(double x, double y, double o[3], void *ud)
{ /* :25-80 — Newton iteration from d3-geo-projection's winkel3 */
    (void)ud;
    if (fabs(y) >= wt_lens_height / 2) return 0;
    if (fabs(x) > wt_artifact_x && fabs(y) > wt_artifact_y) return 0; /* is_inside_artifact_box :93-95 */
    double lambda = x, phi = y;
    const double eps = 0.0001, halfpi = pi / 2;
    for (int iter = 1; iter <= 25; ++iter) {
        double cosphi = cos(phi);
        double sinphi = sin(phi);
        double sin_2phi = sin(2 * phi);
        double sin2phi = sinphi * sinphi;
        double cos2phi = cosphi * cosphi;
        double sinlambda = sin(lambda);
        double coslambda_2 = cos(lambda / 2);
        double sinlambda_2 = sin(lambda / 2);
        double sin2lambda_2 = sinlambda_2 * sinlambda_2;
        double C = 1 - cos2phi * coslambda_2 * coslambda_2;
        double E, F;
        if (C != 0) {
            F = 1 / C;
            E = acos(cosphi * coslambda_2) * sqrt(F);
        } else {
            E = 0;
            F = 0;
        }
        double fx = .5 * (2 * E * cosphi * sinlambda_2 + lambda / halfpi) - x;
        double fy = .5 * (E * sinphi + phi) - y;
        double sigxsiglambda = .5 * F * (cos2phi * sin2lambda_2 + E * cosphi * coslambda_2 * sin2phi) + .5 / halfpi;
        double sigxsigphi = F * (sinlambda * sin_2phi / 4 - E * sinphi * sinlambda_2);
        double sigysiglambda = .125 * F * (sin_2phi * sinlambda_2 - E * sinphi * cos2phi * sinlambda);
        double sigysigphi = .5 * F * (sin2phi * coslambda_2 + E * sin2lambda_2 * cosphi) + .5;
        double denominator = sigxsigphi * sigysiglambda - sigysigphi * sigxsiglambda;
        double siglambda = (fy * sigxsigphi - fx * sigysigphi) / denominator;
        double sigphi = (fx * sigysiglambda - fy * sigxsiglambda) / denominator;
        lambda = lambda - siglambda;
        phi = phi - sigphi;
        if (fabs(siglambda) < eps && fabs(sigphi) < eps) break;
    }
    double lat = phi, lon = lambda;
    double r[3], x0, y0;
    orc_lua_latlon_to_ray(lat, pi, r); /* :75 lens_forward(latlon_to_ray(lat, pi)): the edge of the map at this latitude */
    winkeltripel_forward(r[0], r[1], r[2], &x0, &y0, 0);
    if (fabs(x) < fabs(x0)) {
        orc_lua_latlon_to_ray(lat, lon, o);
        return 1;
    }
    return 0;
}

static void wt_onload(void)
{ /* :82-92 (chunk level) */
    double r[3], x, y;
    orc_lua_latlon_to_ray(pi / 2, 0, r);
    winkeltripel_forward(r[0], r[1], r[2], &x, &y, 0);
    wt_lens_height = 2 * y;
    orc_lua_latlon_to_ray(0, pi, r);
    winkeltripel_forward(r[0], r[1], r[2], &x, &y, 0);
    wt_lens_width = 2 * x;
    wt_artifact_x = wt_lens_width / 2 * 0.71;
    wt_artifact_y = wt_lens_height / 2 * 0.81;
}

/* ---- lenses/eckert4.lua ---------------------------------------------------- */
static double eckert4_solveTheta(double lat)
{ /* :1-11 — 20 Newton steps */
    double t = lat / 2, dt = 0;
    for (int i = 1; i <= 20; ++i) {
        dt = -(t + sin(t) * cos(t) + 2 * sin(t) - (2 + pi * 0.5) * sin(lat)) / (2 * cos(t) * (1 + cos(t)));
        t = t + dt;
    }
    return t;
}

static double eckert4_maxy; /* :43 */

static int eckert4_inverse(double x, double y, double o[3], void *ud)
{ /* :22-31.  get_max_x (:13-20) caches maxx per value of y in script-level variables; maxx is a function of
   * y alone (lat is), so computing it every time gives the same bits */
    (void)ud;
    double t = asin(y / 2 * sqrt((4 + pi) / pi));
    double lat = asin((t + sin(t) * cos(t) + 2 * sin(t)) / (2 + pi * 0.5));
    double lon = sqrt(pi * (4 + pi)) * x / (2 * (1 + cos(t)));
    if (fabs(y) > eckert4_maxy) return 0;
    {
        double tt = eckert4_solveTheta(fabs(lat));
        double maxx = 2 / sqrt(pi * (4 + pi)) * pi * (1 + cos(tt));
        if (fabs(x) > maxx) return 0;
    }
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int eckert4_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :33-39 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    double t = eckert4_solveTheta(lat);
    *ox = 2 / sqrt(pi * (4 + pi)) * lon * (1 + cos(t));
    *oy = 2 * sqrt(pi / (4 + pi)) * sin(t);
    return 1;
}

/* ---- lenses/miller.lua ------------------------------------------------------ */
static double miller_maxy(void) { return 1.25 * log(tan(0.25 * pi + 0.4 * pi * 0.5)); } /* :1 */

static int miller_inverse(double x, double y, double o[3], void *ud)
{ /* :11-18 */
    (void)ud;
    if (fabs(y) > miller_maxy() || fabs(x) > pi) return 0;
    double lon = x;
    double lat = 5.0 / 4 * atan(sinh(4.0 / 5 * y));
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int miller_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :20-25 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon;
    *oy = 1.25 * log(tan(0.25 * pi + 0.4 * lat));
    return 1;
}

/* ---- lenses/gallstereo.lua -------------------------------------------------- */
static const double gs_YF = 1.70710678118654752440, gs_XF = 0.70710678118654752440; /* :1-4 */
static const double gs_RYF = 0.58578643762690495119, gs_RXF = 1.41421356237309504880;

static int gallstereo_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :17-25 — the bounds test is on the ray's components, as written */
    (void)ud;
    const double maxx = gs_XF * pi, maxy = gs_YF * tan(0.5 * pi / 2);
    if (fabs(x) > maxx || fabs(y) > maxy) return 0;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = gs_XF * lon;
    *oy = gs_YF * tan(0.5 * lat);
    return 1;
}

static int gallstereo_inverse(double x, double y, double o[3], void *ud)
{ /* :27-31 */
    (void)ud;
    double lon = gs_RXF * x;
    double lat = 2 * atan(y * gs_RYF);
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

/* ---- lenses/fahey.lua -------------------------------------------------------- */
static int fahey_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :12-18 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    double xx = tan(0.5 * lat);
    double yy = 1.819152 * xx;
    xx = 0.819152 * lon * sqrt(1 - xx * xx);
    *ox = xx;
    *oy = yy;
    return 1;
}

static int fahey_inverse(double x, double y, double o[3], void *ud)
{ /* :20-29 */
    (void)ud;
    const double XR = 0.819152 * pi, YR = 1.819152; /* :1-2 */
    if (x * x / (XR * XR) + y * y / (YR * YR) >= 1) return 0;
    y = y / 1.819152;
    double lat = 2 * atan(y);
    y = 1 - y * y;
    double lon = x / (0.819152 * sqrt(y));
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

/* ---- forward-only lenses ------------------------------------------------------ */
static int eckert1_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* eckert1.lua:15-20 */
    (void)ud;
    const double FC = 0.92131773192356127802, RP = 0.31830988618379067154;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = FC * lon * (1 - RP * fabs(lat));
    *oy = FC * lat;
    return 1;
}

static int eckert5_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* eckert5.lua:10-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon * (1 + cos(lat)) / 2;
    *oy = lat;
    return 1;
}

static int kavrayskiy7_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* kavrayskiy7.lua:10-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = 3 * lon / (2 * pi) * sqrt(pi * pi / 3 - lat * lat);
    *oy = lat;
    return 1;
}

static int winkel2_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* winkel2.lua:10-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon / 2 * (2 / pi + sqrt(pi * pi - 4 * lat * lat) / pi);
    *oy = lat;
    return 1;
}

static int wagner6_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* wagner6.lua:10-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = lon * sqrt(1 - 3 * lat * lat / (pi * pi));
    *oy = lat;
    return 1;
}

static int larrivee_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* larrivee.lua:10-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    *ox = (0.5 + 0.5 * sqrt(cos(lat))) * lon;
    *oy = lat / (cos(lat / 2) * cos(lon / 6));
    return 1;
}

static int gins8_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* gins8.lua:10-20 */
    (void)ud;
    const double Cl = 0.000952426, Cp = 0.162388, C12 = 0.08333333333333333;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    double t = lat * lat;
    double yy = lat * (1 + t * C12);
    double xx = lon * (1 - Cp * t);
    t = lon * lon;
    xx = xx * (0.87 - Cl * t * t);
    *ox = xx;
    *oy = yy;
    return 1;
}

/* ---- lenses/cubestereo.lua -------------------------------------------------- */
static int cubestereo_forward(double rx, double ry, double rz, double *ox, double *oy, void *ud)
{ /* projectcube :6-19, lens_forward :21-24 */
    (void)ud;
    double magx = fabs(rx), magy = fabs(ry), magz = fabs(rz);
    double mag = magz;
    if (magx >= magy && magx >= magz) mag = magx;
    else if (magy >= magx && magy >= magz) mag = magy;
    double x = rx / mag, y = ry / mag, z = rz / mag;
    *ox = x / (z + 1) * 2;
    *oy = y / (z + 1) * 2;
    return 1;
}

static int cubestereo_inverse(double x, double y, double o[3], void *ud)
{ /* :26-50 — returns the ray itself, not latlon_to_ray() */
    (void)ud;
    double rx, ry, rz;
    double magx = fabs(x), magy = fabs(y), z = 2;
    if (magx <= 1 && magy <= 1) {
        rx = x;
        ry = y;
        rz = z - 1;
    } else if (magx > magy) {
        rx = x / magx;
        ry = y / magx;
        rz = z / magx - 1;
    } else {
        rx = x / magy;
        ry = y / magy;
        rz = z / magy - 1;
    }
    double len = sqrt(rx * rx + ry * ry + rz * rz);
    o[0] = rx / len;
    o[1] = ry / len;
    o[2] = rz / len;
    return 1;
}

/* ---- lenses/debug.lua --------------------------------------------------------
 * The one lens that reads `numplates` and calls plate_to_ray: `ud` is the globe (orc_globe *), and
 * orc_debug_lens() must have been called with its numplates (the script's chunk-level code, :1-17). */
static int debug_rows = 1;
static double debug_cols[2] = {0, 0};

int orc_debug_lens(int numplates, orc_lens_def *out)
{
    if (numplates == 4) { debug_rows = 2; debug_cols[0] = 2; debug_cols[1] = 2; }
    else if (numplates == 5) { debug_rows = 2; debug_cols[0] = 3; debug_cols[1] = 2; }
    else if (numplates == 6) { debug_rows = 2; debug_cols[0] = 3; debug_cols[1] = 3; }
    else { debug_rows = 1; debug_cols[0] = numplates; debug_cols[1] = 0; }
    double maxcols = debug_cols[0];                              /* math.max(table.unpack(cols)) */
    if (debug_rows == 2 && debug_cols[1] > maxcols) maxcols = debug_cols[1];
    out->lens_width = maxcols;
    out->lens_height = debug_rows;
    return 1;
}

static int debug_inverse(double x, double y, double o[3], void *ud)
{ /* row :31-38, col :22-29, lens_inverse :40-57 */
    if (!ud) return -1;
    double ny = -y + debug_rows / 2.0; /* rows/2: Lua numbers are doubles */
    double r, v = modf(ny, &r);
    if (ny < 0 || ny >= debug_rows) return 0;
    double rowcols = debug_cols[(int)r];
    double nx = x + rowcols / 2;
    double c, u = modf(nx, &c);
    if (nx < 0 || nx >= rowcols) return 0;
    double plate = c;
    for (double i = 0; i < r; i = i + 1) plate = plate + debug_cols[(int)i];
    return orc_lua_plate_to_ray((const orc_globe *)ud, plate, u, v, o) ? 1 : 0;
}

/* ---- lenses/polyconic.lua --------------------------------------------------- */
static int polyconic_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :7-15 */
    (void)ud;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    if (lat == 0) {
        *ox = lon;
        *oy = 0;
        return 1;
    }
    *ox = 1 / tan(lat) * sin(lon * sin(lat));
    *oy = lat + 1 / tan(lat) * (1 - cos(lon * sin(lat)));
    return 1;
}

/* ---- lenses/gumby.lua -------------------------------------------------------- */
static const double gumby_d = 1, gumbyScale = 0.75; /* :1-2 */

static int gumby_inverse(double x, double y, double o[3], void *ud)
{ /* :10-20 */
    (void)ud;
    const double d = gumby_d, gumbyScaleInv = 1.0 / gumbyScale; /* :3 */
    double k = x * x / ((d + 1) * (d + 1));
    double dscr = k * k * d * d - (k + 1) * (k * d * d - 1);
    double clon = (-k * d + sqrt(dscr)) / (k + 1);
    double S = (d + 1) / (d + clon);
    double lon = atan2(x, S * clon);
    double lat = atan2(y, S);
    lon = lon * gumbyScaleInv;
    lat = lat * gumbyScaleInv;
    orc_lua_latlon_to_ray(lat, lon, o);
    return 1;
}

static int gumby_forward(double x, double y, double z, double *ox, double *oy, void *ud)
{ /* :22-30 */
    (void)ud;
    const double d = gumby_d;
    double lat, lon;
    orc_lua_ray_to_latlon(x, y, z, &lat, &lon);
    lon = lon * gumbyScale;
    lat = lat * gumbyScale;
    double S = (d + 1) / (d + cos(lon));
    *ox = S * sin(lon);
    *oy = S * tan(lat);
    return 1;
}

int orc_find_lens(const char *name, orc_lens_def *out)
{
    memset(out, 0, sizeof *out);
    out->name = name;
    if (!strcmp(name, "panini")) {
        out->inverse = panini_inverse; out->forward = panini_forward;
        out->max_fov = 360; out->max_vfov = 180; out->onload = "f_fov 180";
    } else if (!strcmp(name, "stereographic")) {
        out->inverse = stereographic_inverse; out->forward = stereographic_forward;
        out->max_fov = 360; out->max_vfov = 360; out->onload = "f_fov 180";
    } else if (!strcmp(name, "rectilinear")) {
        out->inverse = rectilinear_inverse; out->forward = rectilinear_forward;
        out->max_fov = 180; out->max_vfov = 180; out->onload = "f_fov 110";
    } else if (!strcmp(name, "equirect")) {
        out->inverse = equirect_inverse; out->forward = equirect_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 2 * pi; out->lens_height = pi; out->onload = "f_contain";
    } else if (!strcmp(name, "cylinder")) {
        out->inverse = cylinder_inverse; out->forward = cylinder_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 2 * pi; out->onload = "f_cover";
    } else if (!strcmp(name, "mercator")) {
        out->inverse = mercator_inverse; out->forward = mercator_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 2 * pi; out->onload = "f_cover";
    } else if (!strcmp(name, "hammer")) {
        out->inverse = hammer_inverse; out->forward = hammer_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = 2 * sqrt(2) * 2; out->lens_height = sqrt(2) * 2; out->onload = "f_contain";
    } else if (!strcmp(name, "fisheye1")) {
        out->inverse = fisheye1_inverse; out->forward = fisheye1_forward;
        out->max_fov = 360; out->max_vfov = 360; out->lens_width = 2 * pi; out->lens_height = 2 * pi; out->onload = "f_contain";
    } else if (!strcmp(name, "mollweide")) {
        out->inverse = mollweide_inverse; out->forward = mollweide_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = 2 * sqrt(2) * 2; out->lens_height = sqrt(2) * 2; out->onload = "f_contain";
    } else if (!strcmp(name, "vandergrinten")) {
        out->inverse = vandergrinten_inverse; out->forward = vandergrinten_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = 2 * vandergrinten_maxr(); out->lens_height = 2 * vandergrinten_maxr(); out->onload = "f_contain";
    } else if (!strcmp(name, "cube")) {
        out->inverse = cube_inverse; out->forward = cube_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 4; out->lens_height = 3; out->onload = "f_contain";
    } else if (!strcmp(name, "winkeltripel")) {
        wt_onload();
        out->inverse = winkeltripel_inverse; out->forward = winkeltripel_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = wt_lens_width; out->lens_height = wt_lens_height; out->onload = "f_contain";
    } else if (!strcmp(name, "eckert4")) {
        double t = eckert4_solveTheta(pi * 0.5); /* :42-50 */
        eckert4_maxy = 2 * sqrt(pi / (4 + pi)) * sin(t);
        t = eckert4_solveTheta(0);
        out->inverse = eckert4_inverse; out->forward = eckert4_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = 2 / sqrt(pi * (4 + pi)) * pi * (1 + cos(t)) * 2; out->lens_height = 2 * eckert4_maxy; out->onload = "f_contain";
    } else if (!strcmp(name, "miller")) {
        out->inverse = miller_inverse; out->forward = miller_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 2 * pi; out->lens_height = miller_maxy() * 2; out->onload = "f_contain";
    } else if (!strcmp(name, "gallstereo")) {
        out->inverse = gallstereo_inverse; out->forward = gallstereo_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = gs_XF * pi * 2; out->lens_height = gs_YF * tan(0.5 * pi / 2) * 2; out->onload = "f_contain";
    } else if (!strcmp(name, "fahey")) {
        out->inverse = fahey_inverse; out->forward = fahey_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 0.819152 * pi * 2; out->lens_height = 1.819152 * 2; out->onload = "f_contain";
    } else if (!strcmp(name, "eckert1")) {
        out->forward = eckert1_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = 0.92131773192356127802 * pi * 2; out->lens_height = 0.92131773192356127802 * pi; out->onload = "f_contain";
    } else if (!strcmp(name, "eckert5")) {
        out->forward = eckert5_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = pi * 2; out->lens_height = pi; out->onload = "f_contain";
    } else if (!strcmp(name, "kavrayskiy7")) {
        out->forward = kavrayskiy7_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 3 * pi / (2 * pi) * sqrt(pi * pi / 3) * 2; out->lens_height = pi; out->onload = "f_contain";
    } else if (!strcmp(name, "winkel2")) {
        out->forward = winkel2_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = pi / 2 * (2 / pi + 1) * 2; out->lens_height = pi; out->onload = "f_contain";
    } else if (!strcmp(name, "wagner6")) {
        out->forward = wagner6_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = pi * 2; out->lens_height = pi; out->onload = "f_contain";
    } else if (!strcmp(name, "larrivee")) {
        out->forward = larrivee_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 2 * pi; out->lens_height = pi / 2 / cos(pi / 2 / 2) * 2; out->onload = "f_contain";
    } else if (!strcmp(name, "gins8")) {
        double r[3], x, y;
        out->forward = gins8_forward;
        out->max_fov = 360; out->max_vfov = 180; out->onload = "f_contain";
        orc_lua_latlon_to_ray(0, pi, r);   /* :22-25 (chunk level) */
        gins8_forward(r[0], r[1], r[2], &x, &y, 0);
        out->lens_width = 2 * fabs(x);
        orc_lua_latlon_to_ray(pi / 2, 0, r);
        gins8_forward(r[0], r[1], r[2], &x, &y, 0);
        out->lens_height = 2 * fabs(y);
    } else if (!strcmp(name, "debug")) {
        out->inverse = debug_inverse;   /* + orc_debug_lens(numplates) for the size; ud = the globe */
        out->onload = "f_contain";
    } else if (!strcmp(name, "cubestereo")) {
        out->inverse = cubestereo_inverse; out->forward = cubestereo_forward;
        out->max_fov = 270; out->max_vfov = 270; out->onload = "f_fov 180";
    } else if (!strcmp(name, "polyconic")) {
        out->forward = polyconic_forward;
        out->max_fov = 360; out->max_vfov = 180; out->onload = "f_fov 360";
    } else if (!strcmp(name, "gumby")) {
        double r[3], x, y;
        out->inverse = gumby_inverse; out->forward = gumby_forward;
        out->max_fov = 360; out->max_vfov = 180; out->onload = "f_contain";
        orc_lua_latlon_to_ray(pi / 2, 0, r);   /* :32-36 (chunk level) */
        gumby_forward(r[0], r[1], r[2], &x, &y, 0);
        out->lens_height = y * 2;
        orc_lua_latlon_to_ray(0, pi, r);
        gumby_forward(r[0], r[1], r[2], &x, &y, 0);
        out->lens_width = x * 2;
    } else if (!strcmp(name, "fisheye2")) {
        double maxr = 2 * sin(pi * 0.5);
        out->inverse = fisheye2_inverse; out->forward = fisheye2_forward;
        out->max_fov = 360; out->max_vfov = 360; out->lens_width = maxr * 2; out->lens_height = maxr * 2; out->onload = "f_contain";
    } else if (!strcmp(name, "quincuncial")) {
        double sqrt2 = sqrt(2);
        out->inverse = quincuncial_inverse;
        out->lens_width = 2 * sqrt2; out->lens_height = 2 * sqrt2; out->onload = "f_contain";
    } else if (!strcmp(name, "sinusoidal")) {
        out->forward = sinusoidal_forward;
        out->max_fov = 360; out->max_vfov = 180; out->lens_width = 2 * pi; out->lens_height = pi; out->onload = "f_contain";
    } else if (!strcmp(name, "winkel1")) {
        out->forward = winkel1_forward;
        out->max_fov = 360; out->max_vfov = 180;
        out->lens_width = pi * (2 / pi + 1) / 2 * 2; out->lens_height = pi; out->onload = "f_contain";
    } else {
        return 0;
    }
    return 1;
}

/* ---- globes ------------------------------------------------------------------ */
static void set_plate(orc_globe *g, int i, double fx, double fy, double fz, double ux, double uy, double uz, double fov)
{
    double f[3] = {fx, fy, fz}, u[3] = {ux, uy, uz};
    orc_globe_set_plate(g, i, f, u, fov);
}

static const double kCube[6][6] = {
    /* globes/cube.lua:3-10 forward, up */
    {0, 0, 1, 0, 1, 0}, {1, 0, 0, 0, 1, 0}, {-1, 0, 0, 0, 1, 0},
    {0, 0, -1, 0, 1, 0}, {0, 1, 0, 0, 0, -1}, {0, -1, 0, 0, 0, 1},
};

/* globes/fast.lua:10-27 */
static int fast_globe_plate(double x, double y, double z, int *plate, void *ud)
{
    (void)ud;
    double big_fov = 160;
    if (z <= 0) return 0; /* return nil */
    double dist = 0.5 / tan(big_fov * pi / 180 / 2);
    double size = 2 * dist * tan(pi / 4);
    double u = x / z * dist;
    double v = y / z * dist;
    if (fabs(u) < size / 2 && fabs(v) < size / 2) *plate = 0; /* small */
    else *plate = 1;                                        /* big */
    return 1;
}

int orc_load_globe(const char *name, orc_globe *g)
{
    int ps = g->platesize;
    memset(g, 0, sizeof *g);
    g->platesize = ps;
    if (!strcmp(name, "cube") || !strcmp(name, "cube_edge") || !strcmp(name, "cube_corner")) {
        int corner = !strcmp(name, "cube_corner"), edge = !strcmp(name, "cube_edge");
        g->numplates = 6;
        for (int i = 0; i < 6; i++) {
            double p[2][3] = {{kCube[i][0], kCube[i][1], kCube[i][2]}, {kCube[i][3], kCube[i][4], kCube[i][5]}};
            if (corner || edge) { /* cube_edge.lua:16-32, cube_corner.lua:16-40 */
                double a = pi / 4;
                for (int k = 0; k < 2; k++) {
                    double x = p[k][0], z = p[k][2];
                    p[k][0] = x * cos(a) - z * sin(a);
                    p[k][2] = x * sin(a) + z * cos(a);
                    if (corner) {
                        double y = p[k][1];
                        z = p[k][2];
                        p[k][1] = y * cos(a) - z * sin(a);
                        p[k][2] = y * sin(a) + z * cos(a);
                    }
                }
            }
            orc_globe_set_plate(g, i, p[0], p[1], 90);
        }
        return 1;
    }
    if (!strcmp(name, "trism")) { /* globes/trism.lua:2-8 */
        g->numplates = 5;
        set_plate(g, 0, -cos(pi / 6), 0, sin(pi / 6), 0, 1, 0, 120);
        set_plate(g, 1, cos(pi / 6), 0, sin(pi / 6), 0, 1, 0, 120);
        set_plate(g, 2, 0, 0, -1, 0, 1, 0, 120);
        set_plate(g, 3, 0, 1, 0, 0, 0, -1, 128);
        set_plate(g, 4, 0, -1, 0, 0, 0, -1, 128);
        return 1;
    }
    if (!strcmp(name, "tetra")) { /* globes/tetra.lua:2-42 */
        double tau = pi * 2; /* fisheye.c:1247 */
        double d120 = tau / 3;
        double d60 = d120 / 2;
        double r = 1;
        double s = 2 * r * sin(d60);
        double h = sqrt(s * s - r * r);
        double theta = acos(r / s);
        double c = s / 2 / sin(theta);
        double e = r * cos(d60);
        double f = h - c;
        double fovr = 2 * atan(r / f);
        double fovd = fovr * 180 / pi + 1;
        double y = e - e * e / (r + e);
        double z = -f + h * e / (r + e);
        g->numplates = 4;
        set_plate(g, 0, 0, -y / f, z / f, 0, -(e - y) / e, (-f - z) / e, fovd);
        set_plate(g, 1, y / f * sin(d120), -y / f * cos(d120), z / f, (e - y) / e * sin(d120), -(e - y) / e * cos(d120), (-f - z) / e, fovd);
        set_plate(g, 2, y / f * sin(-d120), -y / f * cos(-d120), z / f, (e - y) / e * sin(-d120), -(e - y) / e * cos(-d120), (-f - z) / e, fovd);
        set_plate(g, 3, 0, 0, -1, 0, -1, 0, fovd);
        return 1;
    }
    if (!strcmp(name, "fast")) { /* globes/fast.lua:1-8 */
        g->numplates = 2;
        set_plate(g, 0, 0, 0, 1, 0, 1, 0, 90);
        set_plate(g, 1, 0, 0, 1, 0, 1, 0, 160);
        g->plate_fn = fast_globe_plate;
        return 1;
    }
    return 0;
}
