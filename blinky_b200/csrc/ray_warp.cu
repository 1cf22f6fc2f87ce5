// The warp from a ray field turned by a per-frame matrix (blinky_warp_device_rays): each pixel's texel is computed on
// the fly from its view ray, so a head-tracked look-around needs no lensmap, plan or install per frame — only the
// matrix changes.  Frame f of the output equals blinky_set_raymap of the field turned by M_f followed by a one-frame
// blinky_warp_device_view (ray_texel.h holds the per-ray arithmetic).  The supersampled warp
// (blinky_warp_device_rays_supersampled, ray_supersample_kernel) writes each RGBA pixel as the rounded mean of the
// colours of k x k such rays; the bilinear warp (blinky_warp_device_rays_bilinear, ray_bilinear_kernel) the mean of k x k
// bilinear samples, each four texels' colours weighted by where the ray falls between their centres; the trilinear warp
// (blinky_warp_device_rays_trilinear, the pyramid kernels and ray_trilinear_kernel) builds each frame's RGBA mip pyramid
// in the caller's scratch and blends, per pixel, bilinear colours of the two levels around its footprint.
//
// Compiled with --fmad=false: the turn and the globe's float / double arithmetic must round operation by operation
// as the host's -ffp-contract=off build does.
#include "ray_warp.h"

#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>

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

// --------------------------------------------------------------------------
// Trilinear RGBA (blinky_warp_device_rays_trilinear): per frame an RGBA mip pyramid of every plate of the globe in the
// caller's scratch (levels 1..lmax, ray_pyramid_levels' layout), then one sample per pixel blended from two levels.
// --------------------------------------------------------------------------
struct RayPyramidParams {
    uint8_t *scratch;           // frame 0's pyramid
    size_t stride;              // bytes between frames' pyramids (B)
    int lmax;
    uint32_t size[kRayMaxLevels];
    uint64_t off[kRayMaxLevels];
};

// per byte, alpha included: (a + b + c + d + 2) >> 2, in two SWAR words of 16-bit lanes (4 * 255 + 2 fits)
__device__ __forceinline__ uint32_t avg4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    const uint32_t lo = (a & 0x00ff00ffu) + (b & 0x00ff00ffu) + (c & 0x00ff00ffu) + (d & 0x00ff00ffu) + 0x00020002u;
    const uint32_t hi = ((a >> 8) & 0x00ff00ffu) + ((b >> 8) & 0x00ff00ffu) + ((c >> 8) & 0x00ff00ffu) + ((d >> 8) & 0x00ff00ffu) + 0x00020002u;
    return ((lo >> 2) & 0x00ff00ffu) | (((hi >> 2) & 0x00ff00ffu) << 8);
}

__device__ __forceinline__ uint32_t ld_nc_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// Level 1 from the faces: texel (x, y) of plate blockIdx.y of frame blockIdx.z averages the colours of level-0 texels
// (min(2x + i, ps - 1), min(2y + j, ps - 1)), each the colour the nearest RGBA warp draws for that texel (through the
// plate's LUT when f_rubix is on and the texel is off the grid, then the frame's table).
template <bool RUBIX, bool TABLES>
__global__ void __launch_bounds__(kRayThreads) ray_pyramid_base_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ RayPyramidParams q,
                                                                       const __grid_constant__ LensBuildParams P, const __grid_constant__ FaceLayoutParams lay) {
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
    const uint32_t s = q.size[1], ps = q.size[0];
    const uint32_t t = blockIdx.x * kRayThreads + threadIdx.x;
    if (t >= s * s) return;
    const uint32_t y = t / s, x = t - y * s, plate = blockIdx.y, f = blockIdx.z;
    const uint8_t *faces = p.faces + static_cast<size_t>(f) * p.face_stride + lay.plate_base[plate];
    const uint32_t *table = TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr;
    const uint32_t x0 = 2 * x, x1 = min(2 * x + 1, ps - 1), y0 = 2 * y, y1 = min(2 * y + 1, ps - 1);
    bool col[2] = {false, false}, row[2] = {false, false};
    if (RUBIX) {
        col[0] = ray_on_rubix_line(P, x0);
        col[1] = ray_on_rubix_line(P, x1);
        row[0] = ray_on_rubix_line(P, y0);
        row[1] = ray_on_rubix_line(P, y1);
    }
    uint32_t c[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t tx = k & 1 ? x1 : x0, ty = k & 2 ? y1 : y0;
        uint32_t b = ld_texel(faces + static_cast<size_t>(ty) * lay.rowbytes + tx);
        if (RUBIX && !col[k & 1] && !row[k >> 1]) b = s_lut[plate * 256 + b];
        c[k] = TABLES ? __ldg(table + b) : s_rgba[b];
    }
    uint32_t *out = reinterpret_cast<uint32_t *>(q.scratch + static_cast<size_t>(f) * q.stride + q.off[1]) + (static_cast<size_t>(plate) * s + y) * s + x;
    *out = avg4(c[0], c[1], c[2], c[3]);
}

// Level `level` >= 2 from level - 1, per plate (blockIdx.y) and frame (blockIdx.z), with the same clamped 2 x 2 average.
__global__ void __launch_bounds__(kRayThreads) ray_pyramid_reduce_kernel(const __grid_constant__ RayPyramidParams q, int level) {
    const uint32_t s = q.size[level], sp = q.size[level - 1];
    const uint32_t t = blockIdx.x * kRayThreads + threadIdx.x;
    if (t >= s * s) return;
    const uint32_t y = t / s, x = t - y * s, plate = blockIdx.y;
    uint8_t *frame = q.scratch + static_cast<size_t>(blockIdx.z) * q.stride;
    const uint32_t *src = reinterpret_cast<const uint32_t *>(frame + q.off[level - 1]) + static_cast<size_t>(plate) * sp * sp;
    const uint32_t x0 = 2 * x, x1 = min(2 * x + 1, sp - 1), y0 = 2 * y, y1 = min(2 * y + 1, sp - 1);
    const uint32_t c = avg4(src[y0 * sp + x0], src[y0 * sp + x1], src[y1 * sp + x0], src[y1 * sp + x1]);
    reinterpret_cast<uint32_t *>(frame + q.off[level])[(static_cast<size_t>(plate) * s + y) * s + x] = c;
}

// the blend of the four tap colours 00, 10, 01, 11 with 8-bit weights (ray_bilinear_kernel's arithmetic)
__device__ __forceinline__ uint32_t blend4(const uint32_t cq[4], uint32_t wx, uint32_t wy) {
    const uint32_t top_lo = (cq[0] & 0x00ff00ffu) * (256 - wx) + (cq[1] & 0x00ff00ffu) * wx;
    const uint32_t top_hi = ((cq[0] >> 8) & 0x00ff00ffu) * (256 - wx) + ((cq[1] >> 8) & 0x00ff00ffu) * wx;
    const uint32_t bot_lo = (cq[2] & 0x00ff00ffu) * (256 - wx) + (cq[3] & 0x00ff00ffu) * wx;
    const uint32_t bot_hi = ((cq[2] >> 8) & 0x00ff00ffu) * (256 - wx) + ((cq[3] >> 8) & 0x00ff00ffu) * wx;
    const auto blend = [wy](uint32_t t, uint32_t b) { return (t * (256 - wy) + b * wy + 32768u) >> 16; };
    return blend(top_lo & 0xffffu, bot_lo & 0xffffu) | blend(top_hi & 0xffffu, bot_hi & 0xffffu) << 8 | blend(top_lo >> 16, bot_lo >> 16) << 16 |
           blend(top_hi >> 16, bot_hi >> 16) << 24;
}

// the bilinear colour at (u, v) on level L >= 1 of plate `plate` of a frame's pyramid
__device__ __forceinline__ uint32_t level_colour(const RayPyramidParams &q, const uint8_t *pyr, int L, int plate, double u, double v) {
    const int s = static_cast<int>(q.size[L]);
    int x0, y0, wx, wy;
    ray_bilinear_level(u, v, s, &x0, &y0, &wx, &wy);
    const int tx0 = max(x0, 0), tx1 = min(x0 + 1, s - 1), ty0 = max(y0, 0), ty1 = min(y0 + 1, s - 1);
    const uint32_t *lv = reinterpret_cast<const uint32_t *>(pyr + q.off[L]) + static_cast<size_t>(plate) * s * s;
    const uint32_t cq[4] = {ld_nc_u32(lv + ty0 * s + tx0), ld_nc_u32(lv + ty0 * s + tx1), ld_nc_u32(lv + ty1 * s + tx0), ld_nc_u32(lv + ty1 * s + tx1)};
    return blend4(cq, static_cast<uint32_t>(wx), static_cast<uint32_t>(wy));
}

// One thread per output pixel.  The pixel's ray (field pixel (x, y), turned by M_f) is mapped as ray_bilinear maps a
// sample; its footprint rho is the larger distance, in level-0 texels on its plate, to where the turned rays of field
// pixels (x + 1, y) (else (x - 1, y)) and (x, y + 1) (else (x, y - 1)) project onto that plate (ray_footprint2,
// written out so that a backward neighbour is turned only when the forward one is missing or unusable); ray_level
// gives L and w.  Level 0's colour is ray_bilinear_kernel's at K = 1; level L >= 1's is the same blend on the
// pyramid's grid; the output mixes C_L and C_L+1 by w.  With one field and one matrix for every frame of the thread,
// the plate, (u, v), L, w and the level-0 grid tests are carried.
template <bool RUBIX, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads, 1) ray_trilinear_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ RayPyramidParams q,
                                                                    const __grid_constant__ LensBuildParams P, const __grid_constant__ FaceLayoutParams lay) {
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

    const uint32_t pix = blockIdx.x * kRayThreads + threadIdx.x;   // y * W + x (WarpDevice::warp_rays: W H < 2^31)
    if (pix >= p.nitems) return;
    const uint32_t y = pix / p.width, x = pix - y * p.width;
    const uint32_t height = p.nitems / p.width;
    const size_t out_at = static_cast<size_t>(y) * p.pitch + static_cast<size_t>(x) * 4;
    const int f0 = static_cast<int>(blockIdx.y) * p.frames_per_thread;
    const int f1 = min(p.nframes, f0 + p.frames_per_thread);
    const bool carry = p.ray_floats == 0 && p.xform_floats == 0;   // the sample is the same in every frame
    const int ps = P.platesize;

    bool mapped = false;
    int plate = 0, L = 0, w = 0;
    double u = 0, v = 0;
    uint32_t grid = 0;   // f_rubix, level 0: on-grid bits of columns x0, x0 + 1 (0, 1) and rows y0, y0 + 1 (2, 3)
    for (int f = f0; f < f1; ++f) {
        if (f == f0 || !carry) {
            float M[9] = {};
            if (p.xforms) {
                const float *m = p.xforms + static_cast<size_t>(f) * p.xform_floats;
#pragma unroll
                for (int i = 0; i < 9; ++i) M[i] = __ldg(m + i);
            }
            const float *field = p.rays + static_cast<size_t>(f) * p.ray_floats;
            // the field pixel pixel + d, turned and normalised
            const auto ray_at = [&](uint32_t at, float t[3]) {
                const float *r = field + 3 * static_cast<size_t>(at);
                const float ray[3] = {__ldg(r), __ldg(r + 1), __ldg(r + 2)};
                t[0] = ray[0], t[1] = ray[1], t[2] = ray[2];
                if (p.xforms) turn_ray(M, ray, t);
            };
            float n[3];
            ray_at(pix, n);
            int px, py;
            mapped = ray_texel_uv(P, n, &plate, &px, &py, &u, &v);
            L = 0;
            w = 0;
            if (mapped) {
                double a, b, rx = 0, ry = 0;
                if (ray_plate_project(P, plate, n, &a, &b)) {
                    float t[3];
                    double a1, b1;
                    bool done = false;
                    if (x + 1 < p.width) {
                        ray_at(pix + 1, t);
                        ray_normalize3(t);
                        if (ray_plate_project(P, plate, t, &a1, &b1)) rx = ray_axis_rho2(a, b, a1, b1), done = true;
                    }
                    if (!done && x > 0) {
                        ray_at(pix - 1, t);
                        ray_normalize3(t);
                        if (ray_plate_project(P, plate, t, &a1, &b1)) rx = ray_axis_rho2(a, b, a1, b1);
                    }
                    done = false;
                    if (y + 1 < height) {
                        ray_at(pix + p.width, t);
                        ray_normalize3(t);
                        if (ray_plate_project(P, plate, t, &a1, &b1)) ry = ray_axis_rho2(a, b, a1, b1), done = true;
                    }
                    if (!done && y > 0) {
                        ray_at(pix - p.width, t);
                        ray_normalize3(t);
                        if (ray_plate_project(P, plate, t, &a1, &b1)) ry = ray_axis_rho2(a, b, a1, b1);
                    }
                }
                ray_level(ry > rx ? ry : rx, q.lmax, &L, &w);
                if (RUBIX && L == 0) {
                    int x0, y0, wx, wy;
                    ray_bilinear_level(u, v, ps, &x0, &y0, &wx, &wy);
                    const int tx = max(x0, 0), ty = max(y0, 0), tx1 = min(x0 + 1, ps - 1), ty1 = min(y0 + 1, ps - 1);
                    grid = static_cast<uint32_t>(ray_on_rubix_line(P, tx)) | static_cast<uint32_t>(ray_on_rubix_line(P, tx1)) << 1 |
                           static_cast<uint32_t>(ray_on_rubix_line(P, ty)) << 2 | static_cast<uint32_t>(ray_on_rubix_line(P, ty1)) << 3;
                }
            }
        }
        if (KEEP && !mapped) continue;
        const uint32_t *table = TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr;
        uint32_t c;
        if (mapped) {
            const uint8_t *pyr = q.scratch + static_cast<size_t>(f) * q.stride;
            if (L == 0) {
                int x0, y0, wx, wy;
                ray_bilinear_level(u, v, ps, &x0, &y0, &wx, &wy);
                const int tx = max(x0, 0), ty = max(y0, 0), tx1 = min(x0 + 1, ps - 1), ty1 = min(y0 + 1, ps - 1);
                const uint8_t *base = p.faces + static_cast<size_t>(f) * p.face_stride + lay.plate_base[plate];
                uint32_t bq[4] = {ld_texel(base + static_cast<size_t>(ty) * lay.rowbytes + tx), ld_texel(base + static_cast<size_t>(ty) * lay.rowbytes + tx1),
                                  ld_texel(base + static_cast<size_t>(ty1) * lay.rowbytes + tx), ld_texel(base + static_cast<size_t>(ty1) * lay.rowbytes + tx1)};
                if (RUBIX) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (!((grid >> (k & 1)) & 1u) && !((grid >> (2 + (k >> 1))) & 1u)) bq[k] = s_lut[plate * 256 + bq[k]];
                }
                uint32_t cq[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) cq[k] = TABLES ? __ldg(table + bq[k]) : s_rgba[bq[k]];
                c = blend4(cq, static_cast<uint32_t>(wx), static_cast<uint32_t>(wy));
            } else {
                c = level_colour(q, pyr, L, plate, u, v);
            }
            if (w > 0) {
                const uint32_t c1 = level_colour(q, pyr, L + 1, plate, u, v);
                const uint32_t w1 = static_cast<uint32_t>(w), w0 = 256 - w1;
                const uint32_t lo = (c & 0x00ff00ffu) * w0 + (c1 & 0x00ff00ffu) * w1 + 0x00800080u;
                const uint32_t hi = ((c >> 8) & 0x00ff00ffu) * w0 + ((c1 >> 8) & 0x00ff00ffu) * w1 + 0x00800080u;
                c = ((lo >> 8) & 0x00ff00ffu) | (hi & 0xff00ff00u);
            }
        } else {
            const uint32_t bgb = __ldg(p.bg + pix);
            c = TABLES ? __ldg(table + bgb) : s_rgba[bgb];
        }
        st_cs_u32(p.out + static_cast<size_t>(f) * p.out_stride + out_at, c);
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

// the pyramid of every frame (one launch per level 1..lmax), then the trilinear instance of (rubix, keep, tables):
// 2 x 2 x 2 = 8 instances
template <bool RUBIX, bool KEEP>
void launch_trilinear_tables(const RayWarpLaunch &L, const RayWarpParams &p, const RayPyramidParams &q, dim3 grid, cudaStream_t st) {
    if (L.tables) ray_trilinear_kernel<RUBIX, KEEP, true><<<grid, kRayThreads, 0, st>>>(p, q, L.globe, L.layout);
    else ray_trilinear_kernel<RUBIX, KEEP, false><<<grid, kRayThreads, 0, st>>>(p, q, L.globe, L.layout);
}

template <bool RUBIX>
void launch_trilinear_keep(const RayWarpLaunch &L, const RayWarpParams &p, const RayPyramidParams &q, dim3 grid, cudaStream_t st) {
    if (L.keep) launch_trilinear_tables<RUBIX, true>(L, p, q, grid, st);
    else launch_trilinear_tables<RUBIX, false>(L, p, q, grid, st);
}

template <bool RUBIX>
void launch_pyramid_base(const RayWarpLaunch &L, const RayWarpParams &p, const RayPyramidParams &q, dim3 grid, cudaStream_t st) {
    if (L.tables) ray_pyramid_base_kernel<RUBIX, true><<<grid, kRayThreads, 0, st>>>(p, q, L.globe, L.layout);
    else ray_pyramid_base_kernel<RUBIX, false><<<grid, kRayThreads, 0, st>>>(p, q, L.globe, L.layout);
}

void launch_trilinear(const RayWarpLaunch &L, const RayWarpParams &p, dim3 grid, cudaStream_t st) {
    RayPyramidParams q;
    memset(&q, 0, sizeof q);
    q.scratch = static_cast<uint8_t *>(L.scratch);
    q.stride = L.pyramid_bytes;
    q.lmax = L.lmax;
    for (int l = 0; l <= L.lmax; ++l) {
        q.size[l] = static_cast<uint32_t>(L.level_size[l]);
        q.off[l] = L.level_off[l];
    }
    for (int l = 1; l <= L.lmax; ++l) {
        const uint32_t s = q.size[l];
        const dim3 g((s * s + kRayThreads - 1) / kRayThreads, static_cast<unsigned>(L.globe.numplates), static_cast<unsigned>(L.nframes));
        if (l > 1) ray_pyramid_reduce_kernel<<<g, kRayThreads, 0, st>>>(q, l);
        else if (L.rubix) launch_pyramid_base<true>(L, p, q, g, st);
        else launch_pyramid_base<false>(L, p, q, g, st);
    }
    if (L.rubix) launch_trilinear_keep<true>(L, p, q, grid, st);
    else launch_trilinear_keep<false>(L, p, q, grid, st);
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
    if (L.trilinear) {
        launch_trilinear(L, p, grid, st);
        snprintf(buf, sizeof buf, "ray_trilinear_kernel<rubix=%d,keep=%d,tables=%d> grid=(%u,%u) block=%d frames/thread=%d levels=%d", L.rubix, L.keep,
                 L.tables, grid.x, grid.y, kRayThreads, L.frames_per_thread, L.lmax);
    } else if (L.bilinear) {
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
