// The per-ray arithmetic of a warp from a ray field (ray_warp.cu, blinky_warp_device_rays): a view ray turned by a 3x3
// matrix, then mapped through the current globe exactly as FisheyeHost::set_raymap maps it — normalize3, the plate argmax
// of ray_to_plate_index, ray_to_plate_uv, the texel and its range checks, and on_rubix_grid (fisheye_host.cpp), operation
// by operation, with the globe's values as FisheyeHost::device_params computes them.
//
// This is a second copy of that arithmetic, kept apart from the NVRTC text of lens_device.cu on purpose: the warp
// kernel must run without NVRTC and be capturable on its first call.  Host and device share this header; the CPU tests
// compile it with g++ -ffp-contract=off and pin it to the host path, and ray_warp.cu is compiled with --fmad=false, so
// every float and double operation here is one IEEE-rounded operation on both.
#pragma once

#include <math.h>

#include <cstdint>

#include "face_layout.h"   // BLINKY_HD
#include "lens_device.h"   // LensBuildParams

namespace blinky {

// t = M ray, M row-major: t_k = (M[k][0] x + M[k][1] y) + M[k][2] z, every product and sum rounded to float
BLINKY_HD void turn_ray(const float M[9], const float ray[3], float t[3]) {
    for (int k = 0; k < 3; ++k) t[k] = (M[3 * k] * ray[0] + M[3 * k + 1] * ray[1]) + M[3 * k + 2] * ray[2];
}

BLINKY_HD float ray_dot3(const float a[3], const float b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// normalize3 (VectorNormalize): a zero, NaN or overflowing length leaves what the division gives, as on the host
BLINKY_HD void ray_normalize3(float v[3]) {
    float len = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    len = static_cast<float>(sqrt(static_cast<double>(len)));
    if (len) {
        const float inv = 1 / len;
        v[0] *= inv;
        v[1] *= inv;
        v[2] *= inv;
    }
}

// The plate and texel set_raymap gives the unnormalised ray (normalised here, in place) on plates of P.platesize
// texels, with the continuous plate coordinates (u, v) the texel truncates: false when the ray maps to nothing.  The
// plate is the argmax over the globe's P.numplates plates (strict: the lowest index wins ties, NaN never wins).
BLINKY_HD bool ray_texel_uv(const LensBuildParams &P, float ray[3], int *plate, int *px, int *py, double *pu, double *pv) {
    ray_normalize3(ray);
    int best = 0;
    double best_dp = -2;
    for (int i = 0; i < P.numplates; ++i) {
        const double dp = ray_dot3(ray, P.plates[i].forward);   // float dot product, widened
        if (dp > best_dp) {
            best_dp = dp;
            best = i;
        }
    }
    const LensBuildParams::PlateF &p = P.plates[best];
    const double x = ray_dot3(p.right, ray);
    const double y = ray_dot3(p.up, ray);
    const double z = ray_dot3(p.forward, ray);
    const double u = x / z * P.uv_dist[best] + 0.5;
    const double v = -y / z * P.uv_dist[best] + 0.5;
    if (!(u >= 0 && u <= 1 && v >= 0 && v <= 1)) return false;
    const int ps = P.platesize;
    *plate = best;
    *px = static_cast<int>(u * ps);
    *py = static_cast<int>(v * ps);
    *pu = u;
    *pv = v;
    return *px >= 0 && *px < ps && *py >= 0 && *py < ps;
}

// ray_texel_uv without (u, v)
BLINKY_HD bool ray_texel(const LensBuildParams &P, float ray[3], int *plate, int *px, int *py) {
    double u, v;
    return ray_texel_uv(P, ray, plate, px, py, &u, &v);
}

// The bilinear position on a grid of `size` texels per plate side, from the plate coordinates (u, v), in double:
// sx = u * size - 0.5, x0 = floor(sx), wx = (int)((sx - x0) * 256), and likewise y0, wy; the caller clamps the taps
// x0, x0 + 1, y0, y0 + 1 to [0, size - 1].
BLINKY_HD void ray_bilinear_level(double u, double v, int size, int *x0, int *y0, int *wx, int *wy) {
    const double sx = u * size - 0.5, sy = v * size - 0.5;
    const double fx = floor(sx), fy = floor(sy);
    *x0 = static_cast<int>(fx);
    *y0 = static_cast<int>(fy);
    *wx = static_cast<int>((sx - fx) * 256);
    *wy = static_cast<int>((sy - fy) * 256);
}

// The bilinear sample of the unnormalised ray (normalised here, in place; blinky_warp_device_rays_bilinear): mapped
// exactly when ray_texel maps it, on the same plate, at ray_bilinear_level's position on the plate's ps texels.  x0
// and y0 lie in [-1, ps - 1] (u * ps < ps because the texel is in range) and wx, wy in [0, 255] (sx - floor(sx) is
// exact and below 1).
BLINKY_HD bool ray_bilinear(const LensBuildParams &P, float ray[3], int *plate, int *x0, int *y0, int *wx, int *wy) {
    int px, py;
    double u, v;
    if (!ray_texel_uv(P, ray, plate, &px, &py, &u, &v)) return false;
    ray_bilinear_level(u, v, P.platesize, x0, y0, wx, wy);
    return true;
}

// one axis of on_rubix_grid: texel column (or row) t lies in the padding between the rubix cells
BLINKY_HD bool ray_on_rubix_line(const LensBuildParams &P, int t) {
    const double ut = static_cast<double>(t) / P.rubix_unit_px;
    return fmod(ut, P.rubix_block) < P.rubix_pad;
}

// on_rubix_grid: texel (px, py) lies in the padding between the rubix cells, as column px or row py does
BLINKY_HD bool ray_on_rubix_grid(const LensBuildParams &P, int px, int py) { return ray_on_rubix_line(P, px) || ray_on_rubix_line(P, py); }

// ---- trilinear (blinky_warp_device_rays_trilinear, DESIGN §3g) ------------------------------------------------------

// Levels 0..13 at most: set_raymap's plate size limit (6 * ps^2 < 2^28, ps <= 6688) halves to 1 in 13 steps.
constexpr int kRayMaxLevels = 14;

// The mip pyramid of one frame, for plates of ps texels on a globe of nplates plates: size[L] = (size[L-1] + 1) >> 1
// from size[0] = ps down to size[lmax] = 1, and off[L] (L >= 1) the byte offset of level L's plate 0 from the frame's
// pyramid.  Levels 1..lmax are stored level-major, then plate, then rows [size[L]][size[L]] of uint32 texels (level 0
// is the faces themselves); *bytes is their total rounded up to 256.  Returns lmax, or -1 when ps < 1 or the pyramid
// needs more than kRayMaxLevels levels.
BLINKY_HD int ray_pyramid_levels(int ps, int nplates, int size[kRayMaxLevels], uint64_t off[kRayMaxLevels], uint64_t *bytes) {
    if (ps < 1) return -1;
    int lmax = 0;
    uint64_t at = 0;
    size[0] = ps;
    off[0] = 0;
    while (size[lmax] > 1) {
        if (lmax + 1 >= kRayMaxLevels) return -1;
        ++lmax;
        size[lmax] = (size[lmax - 1] + 1) >> 1;
        off[lmax] = at;
        at += 4 * static_cast<uint64_t>(nplates) * static_cast<uint64_t>(size[lmax]) * static_cast<uint64_t>(size[lmax]);
    }
    *bytes = (at + 255) / 256 * 256;
    return lmax;
}

// The projection of the normalised ray n onto plate `plate`, in level-0 texels: x, y, z are the float dot products
// with the plate's right, up and forward, widened to double as in ray_texel_uv.  Usable (true) iff z > 0; then, one
// IEEE double operation each, q = uv_dist * ps / z, a = x * q and b = -y * q.
BLINKY_HD bool ray_plate_project(const LensBuildParams &P, int plate, const float n[3], double *a, double *b) {
    const LensBuildParams::PlateF &p = P.plates[plate];
    const double x = ray_dot3(p.right, n);
    const double y = ray_dot3(p.up, n);
    const double z = ray_dot3(p.forward, n);
    if (!(z > 0)) return false;
    const double q = P.uv_dist[plate] * P.platesize / z;
    *a = x * q;
    *b = -y * q;
    return true;
}

// One axis of the footprint: the squared distance da * da + db * db between the projections (a, b) and (a1, b1).
BLINKY_HD double ray_axis_rho2(double a, double b, double a1, double b1) {
    const double da = a1 - a, db = b1 - b;
    return da * da + db * db;
}

// rho^2, the squared footprint in level-0 texels of a sample on plate `plate` whose normalised ray is n, from the
// normalised (turned) rays of its field neighbours: neighbour(k, t) writes neighbour k — 0: (x + 1, y), 1: (x - 1, y),
// 2: (x, y + 1), 3: (x, y - 1) — to t, or returns false where that field pixel does not exist.  0 when n's own
// projection is not usable.  Per axis: the forward neighbour when it exists and its projection onto the plate is
// usable, else the backward one on the same terms (asked for only then), else the axis gives 0.  rho^2 is the x
// axis's value, replaced by the y axis's when that is greater (so a NaN x axis stays; a NaN y axis is ignored).
template <class Neighbour>
BLINKY_HD double ray_footprint2(const LensBuildParams &P, int plate, const float n[3], const Neighbour &neighbour) {
    double a, b, a1, b1;
    if (!ray_plate_project(P, plate, n, &a, &b)) return 0;
    float t[3];
    double rx = 0, ry = 0;
    if (neighbour(0, t) && ray_plate_project(P, plate, t, &a1, &b1)) rx = ray_axis_rho2(a, b, a1, b1);
    else if (neighbour(1, t) && ray_plate_project(P, plate, t, &a1, &b1)) rx = ray_axis_rho2(a, b, a1, b1);
    if (neighbour(2, t) && ray_plate_project(P, plate, t, &a1, &b1)) ry = ray_axis_rho2(a, b, a1, b1);
    else if (neighbour(3, t) && ray_plate_project(P, plate, t, &a1, &b1)) ry = ray_axis_rho2(a, b, a1, b1);
    return ry > rx ? ry : rx;
}

// ray_footprint2 from neighbour rays already turned and normalised, nullptr where that field pixel does not exist
BLINKY_HD double ray_footprint2(const LensBuildParams &P, int plate, const float n[3], const float *xf, const float *xb, const float *yf,
                                const float *yb) {
    const float *const nb[4] = {xf, xb, yf, yb};
    return ray_footprint2(P, plate, n, [&](int k, float t[3]) {
        if (!nb[k]) return false;
        t[0] = nb[k][0], t[1] = nb[k][1], t[2] = nb[k][2];
        return true;
    });
}

// The level and weight of a footprint, by comparisons only: rho = sqrt(rho2), correctly rounded; *L the largest
// L <= lmax with 2^L <= rho (0 when rho < 1, and for a NaN rho); *w = (int)((rho * 2^-L - 1) * 256) when 1 <= rho
// and L < lmax, else 0 (rho * 2^-L lies in [1, 2) and every step is exact, so w is in 0..255).
BLINKY_HD void ray_level(double rho2, int lmax, int *L, int *w) {
    const double rho = sqrt(rho2);
    int l = 0;
    double p = 1, inv = 1;   // 2^l, 2^-l
    while (l < lmax && 2 * p <= rho) {
        ++l;
        p *= 2;
        inv *= 0.5;
    }
    *L = l;
    *w = rho >= 1 && l < lmax ? static_cast<int>((rho * inv - 1) * 256) : 0;
}

// The packed lensmap entry (BLINKY_LM_*) blinky_set_raymap installs for the ray turned by M (nullptr: the ray as it
// is): a map made in one pass gives an on-grid texel no tint.
BLINKY_HD uint32_t ray_entry(const LensBuildParams &P, const float *M, const float ray[3]) {
    float t[3] = {ray[0], ray[1], ray[2]};
    if (M) turn_ray(M, ray, t);
    int plate, px, py;
    if (!ray_texel(P, t, &plate, &px, &py)) return 7u << 28;
    const uint32_t tint = ray_on_rubix_grid(P, px, py) ? 7u : static_cast<uint32_t>(plate);
    const uint32_t ps = static_cast<uint32_t>(P.platesize);
    return 0x80000000u | tint << 28 | (static_cast<uint32_t>(plate) * ps * ps + static_cast<uint32_t>(px) + static_cast<uint32_t>(py) * ps);
}

}  // namespace blinky
