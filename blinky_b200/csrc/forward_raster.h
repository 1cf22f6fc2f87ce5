// Forward lensmap builder, steps 2-4: the per-thread bodies of the static kernels in
// lens_device.cu, written host/device so that the CPU test-suite can execute them (in any thread
// order) against the serial host builder.  Reference: fisheye.c:2126-2338 (resume_lensmap_forward,
// draw_quad), :1963-1982 (set_lensmap_from_plate), :1922-1960 (rubix grid).
//
// Everything here is integer or IEEE float/double arithmetic in the host's operation order; the
// translation unit that includes it must be compiled without FMA contraction.
#pragma once

#include <cmath>
#include <cstddef>
#include <cstdint>

#include "lens_device.h"

#if defined(__CUDACC__)
#define FWD_HD __host__ __device__ __forceinline__
#else
#define FWD_HD inline
#endif

namespace blinky {

struct FwdPoint {  // screen position of one plate grid point (int2 on the device)
    int x, y;
};
struct FwdMessage {  // one "%d > maxdiff" the reference prints, with the writer key that orders it
    unsigned key, value;
};
constexpr unsigned kFwdMessageCap = 4096;

struct FwdGeom {
    int width, height, ps, numplates;
    double rubix_block, rubix_pad, rubix_unit_px;
    LensBuildParams::PlateF plates[6];
};

struct FwdOut {
    unsigned *idxkey, *tintkey;   // [W*H] highest writer key (+1) overall / among off-grid writers
    unsigned *counters;           // [2] message count, [3..8] display flags
    FwdMessage *messages;
};

FWD_HD unsigned fwd_atomic_max(unsigned *p, unsigned v) {
#if defined(__CUDA_ARCH__)
    return atomicMax(p, v);
#else
    const unsigned o = *p;
    if (v > o) *p = v;
    return o;
#endif
}
FWD_HD unsigned fwd_atomic_inc(unsigned *p) {
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, 1u);
#else
    return (*p)++;
#endif
}

FWD_HD void fwd_apply_patch(FwdPoint *grid, unsigned char *status, const ForwardPatch &pt) {
    status[pt.point] = static_cast<unsigned char>(pt.status);
    if (pt.status == 1) {
        grid[pt.point].x = pt.lx;
        grid[pt.point].y = pt.ly;
    }
}

// The reference keeps two row buffers and `continue`s over nil results (fisheye.c:2151-2189), so a
// nil slot shows whatever the buffer held before: the row two steps earlier, the previous plate's last
// rows at a plate start, zero at the very beginning.  Thread t = (column t/2, buffer t%2) replays its chain.
FWD_HD void fwd_stale_chain(FwdPoint *grid, const unsigned char *status, int ps, int numplates, int t) {
    const int n1 = ps + 1;
    const int i = t >> 1;
    int j = (t & 1) ? ps - 1 : ps;  // buffer `bot` starts with row ps, buffer `top` with row ps-1
    FwdPoint last;
    last.x = last.y = 0;
    for (int p = 0; p < numplates;) {
        const size_t row = (static_cast<size_t>(p) * n1 + j) * n1;
        // slot 1 is skipped together with slot 0 (the `continue` in the px == 0 branch)
        const bool valid = status[row + i] == 1 && !(i == 1 && status[row] != 1);
        if (valid) last = grid[row + i];
        else grid[row + i] = last;
        if (j >= 2) {
            j -= 2;
        } else {
            j = j == 1 ? ps : ps - 1;  // the buffer that ended as `bot` (row 1) takes row ps of the next plate
            ++p;
        }
    }
}

FWD_HD float fwd_dot3(const float *a, const float *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// plate_uv_to_ray (fisheye.c:1198-1214) in the host's float operations (FisheyeHost::plate_uv_to_ray): the
// normalised ray through (u, v) of plate P
FWD_HD void fwd_plate_uv_to_ray(const LensBuildParams::PlateF &P, double u, double v, float r[3]) {
    u -= 0.5;
    v -= 0.5;
    v = -v;
    r[0] = r[1] = r[2] = 0.0f;
    const float fu = static_cast<float>(u), fv = static_cast<float>(v);
    for (int k = 0; k < 3; ++k) r[k] = r[k] + P.dist * P.forward[k];
    for (int k = 0; k < 3; ++k) r[k] = r[k] + fu * P.right[k];
    for (int k = 0; k < 3; ++k) r[k] = r[k] + fv * P.up[k];
    float len = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    len = static_cast<float>(sqrt(static_cast<double>(len)));
    if (len) {
        const float inv = 1 / len;
        r[0] *= inv;
        r[1] *= inv;
        r[2] *= inv;
    }
}

FWD_HD void fwd_set(const FwdGeom &g, const FwdOut &o, int lx, int ly, unsigned key, bool ongrid, int plate) {
    if (lx < 0 || lx >= g.width || ly < 0 || ly >= g.height) return;  // set_lensmap_from_plate's screen check
    o.counters[3 + plate] = 1u;                                         // display flag (benign race: all writers store 1)
    const size_t at = static_cast<size_t>(lx) + static_cast<size_t>(ly) * g.width;
    fwd_atomic_max(&o.idxkey[at], key);
    if (!ongrid) fwd_atomic_max(&o.tintkey[at], key);
}

// a texel owner the host decided (kOwnerPatchOwned | texel)
FWD_HD void fwd_apply_owner_patch(unsigned char *owner, uint32_t patch) {
    owner[patch & ~kOwnerPatchOwned] = (patch & kOwnerPatchOwned) ? kOwnerOwned : 0u;
}

// draw_quad (fisheye.c:2246-2338) for the texel (plate, px, py); key orders the writers like the
// reference's loops do (plate ascending, py descending, px ascending): the highest key wins.
// owner: the owner plane of a globe_plate globe (kOwnerOwned per texel), nullptr for the plate argmax.
FWD_HD void fwd_raster_texel(const FwdGeom &g, const FwdPoint *grid, const FwdOut &o, int plate, int py, int px,
                             const unsigned char *owner = nullptr) {
    const int ps = g.ps, n1 = ps + 1;
    if (owner) {
        if (!(owner[(static_cast<size_t>(plate) * ps + py) * ps + px] & kOwnerOwned)) return;
    } else {
        // the texel belongs to this plate only if the plate wins the ray's argmax (:2193-2199)
        float r[3];
        fwd_plate_uv_to_ray(g.plates[plate], static_cast<double>(px) / ps, static_cast<double>(py) / ps, r);
        int best = 0;
        double best_dp = -2;
        for (int k = 0; k < g.numplates; ++k) {
            const double dp = static_cast<double>(fwd_dot3(r, g.plates[k].forward));
            if (dp > best_dp) {
                best_dp = dp;
                best = k;
            }
        }
        if (best != plate) return;
    }
    const unsigned key = (static_cast<unsigned>(plate) * ps + (ps - 1 - py)) * ps + px + 1u;
    const double ux = static_cast<double>(px) / g.rubix_unit_px, uy = static_cast<double>(py) / g.rubix_unit_px;
    const bool ongrid = fmod(ux, g.rubix_block) < g.rubix_pad || fmod(uy, g.rubix_block) < g.rubix_pad;

    const size_t top = (static_cast<size_t>(plate) * n1 + py) * n1, bot = top + n1;
    const FwdPoint c0 = grid[top + px], c1 = grid[top + px + 1], c2 = grid[bot + px + 1], c3 = grid[bot + px];  // tl, tr, br, bl: clockwise
    const int cx[4] = {c0.x, c1.x, c2.x, c3.x}, cy[4] = {c0.y, c1.y, c2.y, c3.y};
    int x = cx[0], y = cy[0];
    int minx = x, maxx = x, miny = y, maxy = y;
    for (int i = 1; i < 4; ++i) {
        if (cx[i] < minx) minx = cx[i]; else if (cx[i] > maxx) maxx = cx[i];
        if (cy[i] < miny) miny = cy[i]; else if (cy[i] > maxy) maxy = cy[i];
    }
    const int maxdiff = 20;
    // abs() of an int difference, computed like the host does (wraps the same way on overflow)
    const int ddx = static_cast<int>(static_cast<unsigned>(minx) - static_cast<unsigned>(maxx));
    const int ddy = static_cast<int>(static_cast<unsigned>(miny) - static_cast<unsigned>(maxy));
    if ((ddx < 0 ? -ddx : ddx) > maxdiff || (ddy < 0 ? -ddy : ddy) > maxdiff) return;
    if (miny == maxy && minx == maxx) {
        fwd_set(g, o, x, y, key, ongrid, plate);
        return;
    }
    if (miny == maxy) {
        for (int tx = minx; tx <= maxx; ++tx) fwd_set(g, o, tx, miny, key, ongrid, plate);
        return;
    }
    if (minx == maxx) {
        for (int ty = miny; ty <= maxy; ++ty) fwd_set(g, o, x, ty, key, ongrid, plate);
        return;
    }
    for (y = miny; y <= maxy; ++y) {
        int tx[2] = {minx, maxx};
        int found = 0;
        int j = 3;
        for (int i = 0; i < 4; ++i) {
            const int ix = cx[i], iy = cy[i], jx = cx[j], jy = cy[j];
            if ((iy < y && y <= jy) || (jy < y && y <= iy)) {
                const double dy = jy - iy;
                const double dx = jx - ix;
                tx[found] = static_cast<int>(ix + (y - iy) / dy * dx);
                if (++found == 2) break;
            }
            j = i;
        }
        if (tx[0] > tx[1]) {
            const int t = tx[0];
            tx[0] = tx[1];
            tx[1] = t;
        }
        if (tx[1] - tx[0] > maxdiff) {
            const unsigned at = fwd_atomic_inc(&o.counters[2]);
            if (at < kFwdMessageCap) {
                o.messages[at].key = key;
                o.messages[at].value = static_cast<unsigned>(tx[1] - tx[0]);
            }
            return;
        }
        for (x = tx[0]; x <= tx[1]; ++x) fwd_set(g, o, x, y, key, ongrid, plate);
    }
}

FWD_HD void fwd_resolve_pixel(const unsigned *idxkey, const unsigned *tintkey, int32_t *idx, uint8_t *tint, size_t at, int ps) {
    const unsigned k = idxkey[at];
    if (k) {
        const unsigned key = k - 1, px = key % ps, t = key / ps, py = ps - 1 - t % ps, plate = t / ps;
        idx[at] = static_cast<int32_t>(plate * ps * ps + py * ps + px);
    } else {
        idx[at] = -1;
    }
    const unsigned tk = tintkey[at];
    tint[at] = tk ? static_cast<uint8_t>((tk - 1) / ps / ps) : 255;
}

// ---- ray export of a forward lens (DESIGN §3h) -------------------------------------------------------------------

// Where pixel (X, Y) lies in a quad the raster drew it with: (s, t) in [0, 1]^2 with tl = (0, 0), tr = (1, 0),
// br = (1, 1) and bl = (0, 1); cx, cy: the corners in the raster's order {tl, tr, br, bl}.  A corner c came from
// (int)(x / scale + W/2) and the pixel sits at X, so both are measured in half pixels: 2c + 1 and 2X.  The quad is
// split into A = (tl, tr, br) and B = (tl, br, bl); the first non-degenerate triangle that contains the pixel (its
// boundary included) gives (s, t) by exact integer signed areas, one double division each.  When neither contains
// it, the first non-degenerate one does, with s and t clamped.  Both degenerate, or a corner further than the
// raster's maxdiff from tl (corners wrapped at INT_MIN / INT_MAX that its 32-bit bounding box lets through): the
// quad's centre.
FWD_HD void fwd_quad_st(const int cx[4], const int cy[4], int X, int Y, double *s, double *t) {
    *s = *t = 0.5;
    long long qx[4], qy[4];  // corner offsets from tl, in half pixels
    for (int i = 0; i < 4; ++i) {
        const long long dx = static_cast<long long>(cx[i]) - cx[0], dy = static_cast<long long>(cy[i]) - cy[0];
        if (dx > 20 || dx < -20 || dy > 20 || dy < -20) return;
        qx[i] = 2 * dx;
        qy[i] = 2 * dy;
    }
    const long long pxo = 2 * (static_cast<long long>(X) - cx[0]) - 1, pyo = 2 * (static_cast<long long>(Y) - cy[0]) - 1;
    int use = -1;       // the triangle (s, t) comes from: 0 = A, 1 = B
    bool clamp = true;  // it does not contain the pixel
    long long use_a1 = 0, use_a2 = 0, use_area = 0;
    for (int tri = 0; tri < 2 && clamp; ++tri) {
        const int i1 = tri == 0 ? 1 : 2, i2 = tri == 0 ? 2 : 3;  // V0 = tl, V1, V2
        const long long area = qx[i1] * qy[i2] - qy[i1] * qx[i2];
        if (area == 0) continue;
        const long long a1 = pxo * qy[i2] - pyo * qx[i2];  // area(V0, p, V2)
        const long long a2 = qx[i1] * pyo - qy[i1] * pxo;  // area(V0, V1, p)
        const long long a0 = area - a1 - a2;
        const bool inside = area > 0 ? (a0 >= 0 && a1 >= 0 && a2 >= 0) : (a0 <= 0 && a1 <= 0 && a2 <= 0);
        if (use < 0 || inside) {
            use = tri;
            use_a1 = a1;
            use_a2 = a2;
            use_area = area;
        }
        if (inside) clamp = false;
    }
    if (use < 0) return;
    // with l1, l2 the weights of V1, V2: A gives s = l1 + l2, t = l2; B gives s = l1, t = l1 + l2
    const double area = static_cast<double>(use_area);
    double ss = static_cast<double>(use == 0 ? use_a1 + use_a2 : use_a1) / area;
    double tt = static_cast<double>(use == 0 ? use_a2 : use_a1 + use_a2) / area;
    if (clamp) {
        ss = ss < 0 ? 0 : (ss > 1 ? 1 : ss);
        tt = tt < 0 ? 0 : (tt > 1 ? 1 : tt);
    }
    *s = ss;
    *t = tt;
}

// the ray of pixel (X, Y) drawn by the texel (px, py) of plate P through the quad (cx, cy): the plate point at
// ((px - 1/2 + s) / ps, (py - 1/2 + t) / ps), grid point i lying at (i - 1/2) / ps
FWD_HD void fwd_quad_ray(const LensBuildParams::PlateF &P, int ps, int px, int py, const int cx[4], const int cy[4], int X, int Y, float r[3]) {
    double s, t;
    fwd_quad_st(cx, cy, X, Y, &s, &t);
    const double u = ((px - 0.5) + s) / ps, v = ((py - 0.5) + t) / ps;
    fwd_plate_uv_to_ray(P, u, v, r);
}

// the exported ray of pixel (X, Y) from its highest writer key k (idxkey): the zero vector when no texel drew it
FWD_HD void fwd_ray_pixel(const FwdGeom &g, const FwdPoint *grid, unsigned k, int X, int Y, float r[3]) {
    if (!k) {
        r[0] = r[1] = r[2] = 0.0f;
        return;
    }
    const unsigned ps = static_cast<unsigned>(g.ps), key = k - 1, px = key % ps, q = key / ps, py = ps - 1 - q % ps, plate = q / ps;
    const size_t n1 = ps + 1, top = (static_cast<size_t>(plate) * n1 + py) * n1, bot = top + n1;
    const FwdPoint c0 = grid[top + px], c1 = grid[top + px + 1], c2 = grid[bot + px + 1], c3 = grid[bot + px];
    const int cx[4] = {c0.x, c1.x, c2.x, c3.x}, cy[4] = {c0.y, c1.y, c2.y, c3.y};
    fwd_quad_ray(g.plates[plate], g.ps, static_cast<int>(px), static_cast<int>(py), cx, cy, X, Y, r);
}

}  // namespace blinky
