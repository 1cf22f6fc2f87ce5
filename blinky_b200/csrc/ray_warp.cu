// The warp from a ray field turned by a per-frame matrix (blinky_warp_device_rays): each pixel's texel is computed on
// the fly from its view ray, so a head-tracked look-around needs no lensmap, plan or install per frame — only the
// matrix changes.  Frame f of the output equals blinky_set_raymap of the field turned by M_f followed by a one-frame
// blinky_warp_device_view (ray_texel.h holds the per-ray arithmetic).  The supersampled warp
// (blinky_warp_device_rays_supersampled, ray_supersample_kernel) writes each RGBA pixel as the rounded mean of the
// colours of k x k such rays; the bilinear warp (blinky_warp_device_rays_bilinear, ray_bilinear_kernel) the mean of k x k
// bilinear samples, each four texels' colours weighted by where the ray falls between their centres.
//
// Compiled with --fmad=false: the turn and the globe's float / double arithmetic must round operation by operation
// as the host's -ffp-contract=off build does.
#include "ray_warp.h"

#include <cuda_runtime.h>

#include <cstdio>

#include "ray_texel.h"

namespace blinky {

namespace {

constexpr int kRayThreads = 256;

struct RayWarpParams {
    const float *rays;
    size_t ray_floats;          // floats between frames' fields (0: shared)
    const float *xforms;
    size_t xform_floats;        // floats between frames' matrices (0: shared)
    const uint8_t *faces;
    size_t face_stride;
    const uint8_t *bg;
    const uint8_t *lut;
    const uint32_t *rgba;
    size_t table_words;
    uint8_t *out;
    size_t out_stride;
    uint32_t pitch;
    uint32_t width;
    uint32_t nitems;            // quads or pixels
    int nframes;
    int frames_per_thread;
};

__device__ __forceinline__ uint32_t ld_texel(const uint8_t *p) {
    uint32_t v;
    asm volatile("ld.global.nc.u8 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

__device__ __forceinline__ void st_cs_u8(uint8_t *p, uint32_t v) { asm volatile("st.global.cs.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_cs_u32(void *p, uint32_t v) { asm volatile("st.global.cs.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_cs_v4(void *p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// --------------------------------------------------------------------------
// One thread per item: a 4-pixel quad of a row (QUAD, W % 4 == 0) or one pixel.  The thread carries frames
// [blockIdx.y * frames_per_thread, ...): with one shared field it reads its rays once, and with one shared matrix too
// it maps them once; per frame it gathers the texels, tints, expands and stores like warp_gather_kernel (K1) /
// warp_scalar_kernel (K0).  The texel of (plate, px, py) is lay.plate_base[plate] + py * lay.rowbytes + px: dense
// faces are the layout with rowbytes = ps.
// --------------------------------------------------------------------------
template <bool QUAD, bool RUBIX, bool RGBA, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads) ray_warp_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ LensBuildParams P,
                                                               const __grid_constant__ FaceLayoutParams lay) {
    constexpr int NP = QUAD ? 4 : 1;
    __shared__ uint8_t s_lut[RUBIX ? 6 * 256 : 4];
    __shared__ uint32_t s_rgba[RGBA && !TABLES ? 256 : 1];
    if (RUBIX) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.lut);
        uint32_t *dst = reinterpret_cast<uint32_t *>(s_lut);
        for (int i = threadIdx.x; i < 6 * 256 / 4; i += kRayThreads) dst[i] = __ldg(src + i);
    }
    if (RGBA && !TABLES) {
        for (int i = threadIdx.x; i < 256; i += kRayThreads) s_rgba[i] = __ldg(p.rgba + i);
    }
    if (RUBIX || (RGBA && !TABLES)) __syncthreads();

    const uint32_t item = blockIdx.x * kRayThreads + threadIdx.x;
    if (item >= p.nitems) return;
    const uint32_t pix = item * NP;   // dense index y * W + x of the item's first pixel (a quad never straddles rows)
    const uint32_t y = pix / p.width, x = pix - y * p.width;
    const size_t out_at = static_cast<size_t>(y) * p.pitch + static_cast<size_t>(x) * (RGBA ? 4 : 1);
    const int f0 = static_cast<int>(blockIdx.y) * p.frames_per_thread;
    const int f1 = min(p.nframes, f0 + p.frames_per_thread);

    // a pixel's texel, packed: px (bits 0-12), py (13-25), plate (26-28), on the rubix grid (29), mapped (31) —
    // WarpDevice::warp_rays refuses a plate size beyond set_raymap's limit, 6 * ps^2 < 2^28, so ps <= 6688 < 2^13
    constexpr uint32_t kMapped = 0x80000000u, kOnGrid = 0x20000000u;
    float ray[NP][3];
    uint32_t tx[NP];
    uint32_t valid = 0;   // bit k: pixel k is mapped
    for (int f = f0; f < f1; ++f) {
        if (f == f0 || p.ray_floats) {
            const float *r = p.rays + static_cast<size_t>(f) * p.ray_floats + 3 * static_cast<size_t>(pix);
#pragma unroll
            for (int k = 0; k < NP; ++k)
#pragma unroll
                for (int c = 0; c < 3; ++c) ray[k][c] = __ldg(r + 3 * k + c);
        }
        if (f == f0 || p.ray_floats || p.xform_floats) {
            float M[9] = {};
            if (p.xforms) {
                const float *m = p.xforms + static_cast<size_t>(f) * p.xform_floats;
#pragma unroll
                for (int i = 0; i < 9; ++i) M[i] = __ldg(m + i);
            }
            valid = 0;
#pragma unroll
            for (int k = 0; k < NP; ++k) {
                float t[3] = {ray[k][0], ray[k][1], ray[k][2]};
                if (p.xforms) turn_ray(M, ray[k], t);
                int plate = 0, px = 0, py = 0;
                tx[k] = 0;
                if (ray_texel(P, t, &plate, &px, &py)) {
                    valid |= 1u << k;
                    tx[k] = kMapped | static_cast<uint32_t>(plate) << 26 | static_cast<uint32_t>(py) << 13 | static_cast<uint32_t>(px);
                }
            }
            // (the tint is read only with f_rubix: the grid test's two fmods are skipped otherwise)
            if (RUBIX) {
#pragma unroll
                for (int k = 0; k < NP; ++k)
                    if ((tx[k] & kMapped) && ray_on_rubix_grid(P, tx[k] & 0x1fffu, (tx[k] >> 13) & 0x1fffu)) tx[k] |= kOnGrid;
            }
        }
        if (KEEP && valid == 0) continue;
        const uint8_t *faces = p.faces + static_cast<size_t>(f) * p.face_stride;
        const uint32_t *table = RGBA && TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr;
        const bool all_valid = valid == (1u << NP) - 1;
        uint32_t bgw = 0;
        if (!KEEP && !all_valid) bgw = QUAD ? __ldg(reinterpret_cast<const uint32_t *>(p.bg) + item) : __ldg(p.bg + pix);
        uint32_t px4[NP];
#pragma unroll
        for (int k = 0; k < NP; ++k) {
            uint32_t b;
            if (tx[k] & kMapped) {
                const uint32_t plate = (tx[k] >> 26) & 7u;
                b = ld_texel(faces + lay.plate_base[plate] + static_cast<size_t>((tx[k] >> 13) & 0x1fffu) * lay.rowbytes + (tx[k] & 0x1fffu));
                if (RUBIX && !(tx[k] & kOnGrid)) b = s_lut[plate * 256 + b];
            } else {
                b = (bgw >> (8 * k)) & 0xffu;
            }
            if (RGBA) b = TABLES ? __ldg(table + b) : s_rgba[b];
            px4[k] = b;
        }
        uint8_t *o = p.out + static_cast<size_t>(f) * p.out_stride + out_at;
        if (QUAD && !(KEEP && !all_valid)) {
            if (RGBA) st_cs_v4(o, px4[0], px4[NP > 1 ? 1 : 0], px4[NP > 2 ? 2 : 0], px4[NP > 3 ? 3 : 0]);
            else st_cs_u32(o, px4[0] | (px4[NP > 1 ? 1 : 0] << 8) | (px4[NP > 2 ? 2 : 0] << 16) | (px4[NP > 3 ? 3 : 0] << 24));
        } else {
#pragma unroll
            for (int k = 0; k < NP; ++k) {
                if (KEEP && !((valid >> k) & 1u)) continue;
                if (RGBA) st_cs_u32(o + 4 * k, px4[k]);
                else st_cs_u8(o + k, px4[k]);
            }
        }
    }
}

// --------------------------------------------------------------------------
// Supersampled RGBA (blinky_warp_device_rays_supersampled): one thread per output pixel, whose K x K samples are the
// field pixels (K x + i, K y + j) of a dense K W x K H field, each turned and mapped as ray_warp_kernel maps a pixel's
// ray.  Sample j's row is 12 K contiguous bytes of the field, so a warp reads 384 K contiguous bytes per sub-row.  The
// samples' colours are summed in two SWAR words (bytes 0 and 2, bytes 1 and 3, in 16-bit lanes: 16 * 255 fits) and each
// byte written is (sum + K^2 / 2) / K^2.  With one field and one matrix for every frame of the thread, the K^2 packed
// texels are mapped once and carried; otherwise each frame re-reads its rays (a shared field of a small view from the
// caches; at 4K from HBM, which the per-sample arithmetic outweighs).
// (The minimum of one block per SM lets ptxas size the registers to the instance: with the default it held K = 2 with
// f_rubix to 64 registers and spilled.)
// --------------------------------------------------------------------------
template <int K, bool RUBIX, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads, 1) ray_supersample_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ LensBuildParams P,
                                                                      const __grid_constant__ FaceLayoutParams lay) {
    constexpr int S = K * K;
    __shared__ uint8_t s_lut[RUBIX ? 6 * 256 : 4];
    __shared__ uint32_t s_rgba[TABLES ? 1 : 256];
    if (RUBIX) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.lut);
        uint32_t *dst = reinterpret_cast<uint32_t *>(s_lut);
        for (int i = threadIdx.x; i < 6 * 256 / 4; i += kRayThreads) dst[i] = __ldg(src + i);
    }
    if (!TABLES) {
        for (int i = threadIdx.x; i < 256; i += kRayThreads) s_rgba[i] = __ldg(p.rgba + i);
    }
    if (RUBIX || !TABLES) __syncthreads();

    const uint32_t pix = blockIdx.x * kRayThreads + threadIdx.x;   // y * W + x (WarpDevice::warp_rays: K^2 W H < 2^31)
    if (pix >= p.nitems) return;
    const uint32_t y = pix / p.width, x = pix - y * p.width;
    const uint32_t fw = K * p.width;                                // field row, in field pixels
    const uint32_t first = K * y * fw + K * x;                      // field pixel of sample (0, 0)
    const size_t out_at = static_cast<size_t>(y) * p.pitch + static_cast<size_t>(x) * 4;
    const int f0 = static_cast<int>(blockIdx.y) * p.frames_per_thread;
    const int f1 = min(p.nframes, f0 + p.frames_per_thread);
    const bool carry = p.ray_floats == 0 && p.xform_floats == 0;   // the texels are the same in every frame

    // a sample's texel, packed as in ray_warp_kernel: px (bits 0-12), py (13-25), plate (26-28), on the grid (29), mapped (31)
    constexpr uint32_t kMapped = 0x80000000u, kOnGrid = 0x20000000u;
    uint32_t tx[S];
    int mapped = 0;
    for (int f = f0; f < f1; ++f) {
        if (f == f0 || !carry) {
            float M[9] = {};
            if (p.xforms) {
                const float *m = p.xforms + static_cast<size_t>(f) * p.xform_floats;
#pragma unroll
                for (int i = 0; i < 9; ++i) M[i] = __ldg(m + i);
            }
            const float *field = p.rays + static_cast<size_t>(f) * p.ray_floats;
            mapped = 0;
#pragma unroll
            for (int j = 0; j < K; ++j) {
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    const float *r = field + 3 * static_cast<size_t>(first + j * fw + i);
                    const float ray[3] = {__ldg(r), __ldg(r + 1), __ldg(r + 2)};
                    float t[3] = {ray[0], ray[1], ray[2]};
                    if (p.xforms) turn_ray(M, ray, t);
                    int plate = 0, px = 0, py = 0;
                    tx[j * K + i] = 0;
                    if (ray_texel(P, t, &plate, &px, &py)) {
                        ++mapped;
                        tx[j * K + i] = kMapped | static_cast<uint32_t>(plate) << 26 | static_cast<uint32_t>(py) << 13 | static_cast<uint32_t>(px);
                    }
                }
            }
            if (RUBIX) {
#pragma unroll
                for (int s = 0; s < S; ++s)
                    if ((tx[s] & kMapped) && ray_on_rubix_grid(P, tx[s] & 0x1fffu, (tx[s] >> 13) & 0x1fffu)) tx[s] |= kOnGrid;
            }
        }
        if (KEEP && mapped == 0) continue;
        const uint8_t *faces = p.faces + static_cast<size_t>(f) * p.face_stride;
        const uint32_t *table = TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr;
        const uint32_t bgb = mapped < S ? __ldg(p.bg + pix) : 0u;
        uint32_t lo = 0, hi = 0;   // bytes 0 and 2, bytes 1 and 3 of the sum, in 16-bit lanes
#pragma unroll
        for (int s = 0; s < S; ++s) {
            uint32_t b = bgb;
            if (tx[s] & kMapped) {
                const uint32_t plate = (tx[s] >> 26) & 7u;
                b = ld_texel(faces + lay.plate_base[plate] + static_cast<size_t>((tx[s] >> 13) & 0x1fffu) * lay.rowbytes + (tx[s] & 0x1fffu));
                if (RUBIX && !(tx[s] & kOnGrid)) b = s_lut[plate * 256 + b];
            }
            const uint32_t c = TABLES ? __ldg(table + b) : s_rgba[b];
            lo += c & 0x00ff00ffu;
            hi += (c >> 8) & 0x00ff00ffu;
        }
        constexpr uint32_t half = S / 2;
        const uint32_t rgba = ((lo & 0xffffu) + half) / S | (((hi & 0xffffu) + half) / S) << 8 | (((lo >> 16) + half) / S) << 16 |
                              (((hi >> 16) + half) / S) << 24;
        st_cs_u32(p.out + static_cast<size_t>(f) * p.out_stride + out_at, rgba);
    }
}

// --------------------------------------------------------------------------
// Bilinear RGBA (blinky_warp_device_rays_bilinear): one thread per output pixel, whose K x K samples (K = 1..4) are the
// field pixels of ray_supersample_kernel, each turned and mapped as ray_warp_kernel maps a pixel's ray.  A mapped
// sample's colour blends the table colours of its four taps (x0 | x0 + 1, y0 | y0 + 1, clamped to its own plate) with
// the weights of ray_bilinear; an unmapped one is the pixel's background colour; the K^2 colours are averaged as
// ray_supersample_kernel averages them.  With one field and one matrix for every frame of the thread the samples'
// packed positions are mapped once and carried.
// (A minimum of one block per SM, as for ray_supersample_kernel: ptxas sizes the registers to the instance.)
// --------------------------------------------------------------------------
template <int K, bool RUBIX, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads, 1) ray_bilinear_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ LensBuildParams P,
                                                                   const __grid_constant__ FaceLayoutParams lay) {
    constexpr int S = K * K;
    __shared__ uint8_t s_lut[RUBIX ? 6 * 256 : 4];
    __shared__ uint32_t s_rgba[TABLES ? 1 : 256];
    if (RUBIX) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.lut);
        uint32_t *dst = reinterpret_cast<uint32_t *>(s_lut);
        for (int i = threadIdx.x; i < 6 * 256 / 4; i += kRayThreads) dst[i] = __ldg(src + i);
    }
    if (!TABLES) {
        for (int i = threadIdx.x; i < 256; i += kRayThreads) s_rgba[i] = __ldg(p.rgba + i);
    }
    if (RUBIX || !TABLES) __syncthreads();

    const uint32_t pix = blockIdx.x * kRayThreads + threadIdx.x;   // y * W + x (WarpDevice::warp_rays: K^2 W H < 2^31)
    if (pix >= p.nitems) return;
    const uint32_t y = pix / p.width, x = pix - y * p.width;
    const uint32_t fw = K * p.width;                                // field row, in field pixels
    const uint32_t first = K * y * fw + K * x;                      // field pixel of sample (0, 0)
    const size_t out_at = static_cast<size_t>(y) * p.pitch + static_cast<size_t>(x) * 4;
    const int f0 = static_cast<int>(blockIdx.y) * p.frames_per_thread;
    const int f1 = min(p.nframes, f0 + p.frames_per_thread);
    const bool carry = p.ray_floats == 0 && p.xform_floats == 0;   // the samples are the same in every frame
    const int ps = P.platesize;

    // a sample, packed in two words.  pos: the clamped first tap tx (bits 0-12) and ty (13-25), plate (26-28), the
    // second tap's steps dx (29) and dy (30) — 0 where the clamp folds both taps onto one texel — and mapped (31).
    // wt: wx (bits 0-7), wy (8-15), and with f_rubix the grid tests of column tx (16), tx + dx (17), row ty (18) and
    // ty + dy (19).
    constexpr uint32_t kMapped = 0x80000000u, kDx = 0x20000000u, kDy = 0x40000000u;
    uint32_t pos[S], wt[S];
    int mapped = 0;
    for (int f = f0; f < f1; ++f) {
        if (f == f0 || !carry) {
            float M[9] = {};
            if (p.xforms) {
                const float *m = p.xforms + static_cast<size_t>(f) * p.xform_floats;
#pragma unroll
                for (int i = 0; i < 9; ++i) M[i] = __ldg(m + i);
            }
            const float *field = p.rays + static_cast<size_t>(f) * p.ray_floats;
            mapped = 0;
#pragma unroll
            for (int j = 0; j < K; ++j) {
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    const float *r = field + 3 * static_cast<size_t>(first + j * fw + i);
                    const float ray[3] = {__ldg(r), __ldg(r + 1), __ldg(r + 2)};
                    float t[3] = {ray[0], ray[1], ray[2]};
                    if (p.xforms) turn_ray(M, ray, t);
                    int plate = 0, x0 = 0, y0 = 0, wx = 0, wy = 0;
                    pos[j * K + i] = 0;
                    wt[j * K + i] = 0;
                    if (ray_bilinear(P, t, &plate, &x0, &y0, &wx, &wy)) {
                        ++mapped;
                        const uint32_t tx = max(x0, 0), ty = max(y0, 0);
                        const uint32_t dx = x0 >= 0 && x0 < ps - 1, dy = y0 >= 0 && y0 < ps - 1;
                        pos[j * K + i] = kMapped | dy << 30 | dx << 29 | static_cast<uint32_t>(plate) << 26 | ty << 13 | tx;
                        wt[j * K + i] = static_cast<uint32_t>(wy) << 8 | static_cast<uint32_t>(wx);
                    }
                }
            }
            if (RUBIX) {
#pragma unroll
                for (int s = 0; s < S; ++s) {
                    if (!(pos[s] & kMapped)) continue;
                    const int tx = pos[s] & 0x1fffu, ty = (pos[s] >> 13) & 0x1fffu, dx = (pos[s] >> 29) & 1u, dy = (pos[s] >> 30) & 1u;
                    wt[s] |= static_cast<uint32_t>(ray_on_rubix_line(P, tx)) << 16 | static_cast<uint32_t>(ray_on_rubix_line(P, tx + dx)) << 17 |
                             static_cast<uint32_t>(ray_on_rubix_line(P, ty)) << 18 | static_cast<uint32_t>(ray_on_rubix_line(P, ty + dy)) << 19;
                }
            }
        }
        if (KEEP && mapped == 0) continue;
        const uint8_t *faces = p.faces + static_cast<size_t>(f) * p.face_stride;
        const uint32_t *table = TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr;
        const uint32_t bgb = mapped < S ? __ldg(p.bg + pix) : 0u;
        uint32_t lo = 0, hi = 0;   // bytes 0 and 2, bytes 1 and 3 of the sum over the samples, in 16-bit lanes
#pragma unroll
        for (int s = 0; s < S; ++s) {
            uint32_t c;
            if (pos[s] & kMapped) {
                const uint32_t plate = (pos[s] >> 26) & 7u;
                const uint8_t *t00 = faces + lay.plate_base[plate] + static_cast<size_t>((pos[s] >> 13) & 0x1fffu) * lay.rowbytes + (pos[s] & 0x1fffu);
                const uint32_t dx = (pos[s] & kDx) ? 1u : 0u;
                const size_t dy = (pos[s] & kDy) ? lay.rowbytes : 0;
                uint32_t b[4] = {ld_texel(t00), ld_texel(t00 + dx), ld_texel(t00 + dy), ld_texel(t00 + dy + dx)};   // 00, 10, 01, 11
                if (RUBIX) {
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        if (!((wt[s] >> (16 + (q & 1))) & 1u) && !((wt[s] >> (18 + (q >> 1))) & 1u)) b[q] = s_lut[plate * 256 + b[q]];
                }
                uint32_t cq[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) cq[q] = TABLES ? __ldg(table + b[q]) : s_rgba[b[q]];
                const uint32_t wx = wt[s] & 0xffu, wy = (wt[s] >> 8) & 0xffu;
                // horizontal step in 16-bit lanes (255 * 256 fits), the vertical one per byte in 32 bits
                const uint32_t top_lo = (cq[0] & 0x00ff00ffu) * (256 - wx) + (cq[1] & 0x00ff00ffu) * wx;
                const uint32_t top_hi = ((cq[0] >> 8) & 0x00ff00ffu) * (256 - wx) + ((cq[1] >> 8) & 0x00ff00ffu) * wx;
                const uint32_t bot_lo = (cq[2] & 0x00ff00ffu) * (256 - wx) + (cq[3] & 0x00ff00ffu) * wx;
                const uint32_t bot_hi = ((cq[2] >> 8) & 0x00ff00ffu) * (256 - wx) + ((cq[3] >> 8) & 0x00ff00ffu) * wx;
                const auto blend = [wy](uint32_t t, uint32_t b) { return (t * (256 - wy) + b * wy + 32768u) >> 16; };
                c = blend(top_lo & 0xffffu, bot_lo & 0xffffu) | blend(top_hi & 0xffffu, bot_hi & 0xffffu) << 8 | blend(top_lo >> 16, bot_lo >> 16) << 16 |
                    blend(top_hi >> 16, bot_hi >> 16) << 24;
            } else {
                c = TABLES ? __ldg(table + bgb) : s_rgba[bgb];
            }
            if (S == 1) {
                lo = c;
                continue;
            }
            lo += c & 0x00ff00ffu;
            hi += (c >> 8) & 0x00ff00ffu;
        }
        uint32_t rgba = lo;
        if (S > 1) {
            constexpr uint32_t half = S / 2;
            rgba = ((lo & 0xffffu) + half) / S | (((hi & 0xffffu) + half) / S) << 8 | (((lo >> 16) + half) / S) << 16 | (((hi >> 16) + half) / S) << 24;
        }
        st_cs_u32(p.out + static_cast<size_t>(f) * p.out_stride + out_at, rgba);
    }
}

template <bool QUAD, bool RUBIX, bool RGBA, bool KEEP, bool TABLES>
void launch_instance(const RayWarpParams &p, const LensBuildParams &P, const FaceLayoutParams &lay, dim3 grid, cudaStream_t st) {
    ray_warp_kernel<QUAD, RUBIX, RGBA, KEEP, TABLES><<<grid, kRayThreads, 0, st>>>(p, P, lay);
}

// the instance of (quads, rubix, rgba, keep, tables): per-frame tables exist only in RGBA, so 24 instances
template <bool QUAD, bool RUBIX, bool RGBA, bool KEEP>
void launch_tables(bool tables, const RayWarpParams &p, const LensBuildParams &P, const FaceLayoutParams &lay, dim3 grid, cudaStream_t st) {
    if constexpr (RGBA) {
        if (tables) return launch_instance<QUAD, RUBIX, RGBA, KEEP, true>(p, P, lay, grid, st);
    }
    launch_instance<QUAD, RUBIX, RGBA, KEEP, false>(p, P, lay, grid, st);
}

template <bool QUAD, bool RUBIX, bool RGBA>
void launch_keep(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.keep) launch_tables<QUAD, RUBIX, RGBA, true>(L.tables, p, L.globe, L.layout, grid, st);
    else launch_tables<QUAD, RUBIX, RGBA, false>(L.tables, p, L.globe, L.layout, grid, st);
}

template <bool QUAD, bool RUBIX>
void launch_rgba(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.rgba) launch_keep<QUAD, RUBIX, true>(L, p, grid, st);
    else launch_keep<QUAD, RUBIX, false>(L, p, grid, st);
}

template <bool QUAD>
void launch_rubix(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.rubix) launch_rgba<QUAD, true>(L, p, grid, st);
    else launch_rgba<QUAD, false>(L, p, grid, st);
}

// the supersampled instance of (factor, rubix, keep, tables): 3 x 2 x 2 x 2 = 24 instances
template <int K, bool RUBIX, bool KEEP>
void launch_supersample_tables(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.tables) ray_supersample_kernel<K, RUBIX, KEEP, true><<<grid, kRayThreads, 0, st>>>(p, L.globe, L.layout);
    else ray_supersample_kernel<K, RUBIX, KEEP, false><<<grid, kRayThreads, 0, st>>>(p, L.globe, L.layout);
}

template <int K, bool RUBIX>
void launch_supersample_keep(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.keep) launch_supersample_tables<K, RUBIX, true>(L, p, grid, st);
    else launch_supersample_tables<K, RUBIX, false>(L, p, grid, st);
}

template <int K>
void launch_supersample_rubix(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.rubix) launch_supersample_keep<K, true>(L, p, grid, st);
    else launch_supersample_keep<K, false>(L, p, grid, st);
}

void launch_supersample(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.factor == 2) launch_supersample_rubix<2>(L, p, grid, st);
    else if (L.factor == 3) launch_supersample_rubix<3>(L, p, grid, st);
    else launch_supersample_rubix<4>(L, p, grid, st);
}

// the bilinear instance of (factor, rubix, keep, tables): 4 x 2 x 2 x 2 = 32 instances
template <int K, bool RUBIX, bool KEEP>
void launch_bilinear_tables(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.tables) ray_bilinear_kernel<K, RUBIX, KEEP, true><<<grid, kRayThreads, 0, st>>>(p, L.globe, L.layout);
    else ray_bilinear_kernel<K, RUBIX, KEEP, false><<<grid, kRayThreads, 0, st>>>(p, L.globe, L.layout);
}

template <int K, bool RUBIX>
void launch_bilinear_keep(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.keep) launch_bilinear_tables<K, RUBIX, true>(L, p, grid, st);
    else launch_bilinear_tables<K, RUBIX, false>(L, p, grid, st);
}

template <int K>
void launch_bilinear_rubix(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.rubix) launch_bilinear_keep<K, true>(L, p, grid, st);
    else launch_bilinear_keep<K, false>(L, p, grid, st);
}

void launch_bilinear(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    if (L.factor == 1) launch_bilinear_rubix<1>(L, p, grid, st);
    else if (L.factor == 2) launch_bilinear_rubix<2>(L, p, grid, st);
    else if (L.factor == 3) launch_bilinear_rubix<3>(L, p, grid, st);
    else launch_bilinear_rubix<4>(L, p, grid, st);
}

}  // namespace

bool launch_ray_warp(const RayWarpLaunch &L, std::string *name, int *cuda_err) {
    RayWarpParams p;
    p.rays = L.rays;
    p.ray_floats = L.ray_stride / 4;
    p.xforms = L.xforms;
    p.xform_floats = L.xform_stride / 4;
    p.faces = static_cast<const uint8_t *>(L.faces);
    p.face_stride = L.face_stride;
    p.bg = L.bg;
    p.lut = L.lut;
    p.rgba = L.palette;
    p.table_words = L.table_stride / 4;
    p.out = static_cast<uint8_t *>(L.out);
    p.out_stride = L.out_stride;
    p.pitch = L.pitch;
    p.width = static_cast<uint32_t>(L.width);
    const size_t npix = static_cast<size_t>(L.width) * static_cast<size_t>(L.height);
    p.nitems = static_cast<uint32_t>(L.quads ? npix / 4 : npix);   // (supersampled, bilinear: one item per output pixel, never quads)
    p.nframes = L.nframes;
    p.frames_per_thread = L.frames_per_thread;
    const dim3 grid(static_cast<unsigned>((p.nitems + kRayThreads - 1) / kRayThreads),
                    static_cast<unsigned>((L.nframes + L.frames_per_thread - 1) / L.frames_per_thread));
    cudaStream_t st = static_cast<cudaStream_t>(L.stream);
    char buf[192];
    if (L.bilinear) {
        launch_bilinear(L, p, grid, st);
        snprintf(buf, sizeof buf, "ray_bilinear_kernel<k=%d,rubix=%d,keep=%d,tables=%d> grid=(%u,%u) block=%d frames/thread=%d", L.factor, L.rubix,
                 L.keep, L.tables, grid.x, grid.y, kRayThreads, L.frames_per_thread);
    } else if (L.factor > 1) {
        launch_supersample(L, p, grid, st);
        snprintf(buf, sizeof buf, "ray_supersample_kernel<k=%d,rubix=%d,keep=%d,tables=%d> grid=(%u,%u) block=%d frames/thread=%d", L.factor, L.rubix,
                 L.keep, L.tables, grid.x, grid.y, kRayThreads, L.frames_per_thread);
    } else {
        if (L.quads) launch_rubix<true>(L, p, grid, st);
        else launch_rubix<false>(L, p, grid, st);
        snprintf(buf, sizeof buf, "ray_warp_kernel<quad=%d,rubix=%d,rgba=%d,keep=%d,tables=%d> grid=(%u,%u) block=%d frames/thread=%d", L.quads,
                 L.rubix, L.rgba, L.keep, L.tables, grid.x, grid.y, kRayThreads, L.frames_per_thread);
    }
    *name = buf;
    const cudaError_t e = cudaGetLastError();
    *cuda_err = static_cast<int>(e);
    return e == cudaSuccess;
}

}  // namespace blinky
