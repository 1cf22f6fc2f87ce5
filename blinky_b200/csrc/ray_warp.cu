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
#include <type_traits>

#include "ray_texel.h"

namespace blinky {

namespace {

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

// ---- per-sample routines --------------------------------------------------------------------------------------------

// Copies the rubix tint LUTs (RUBIX: [6][256] bytes, as words) and the context's RGBA table (SHARED_TABLE) into the
// CTA's shared memory; every thread calls it before any returns.
template <bool RUBIX, bool SHARED_TABLE>
__device__ __forceinline__ void stage_tables(const RayWarpParams &p, uint32_t *s_lut, uint32_t *s_rgba) {
    if (RUBIX) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.lut);
        for (int i = threadIdx.x; i < 6 * 256 / 4; i += kRayThreads) s_lut[i] = __ldg(src + i);
    }
    if (SHARED_TABLE) {
        for (int i = threadIdx.x; i < 256; i += kRayThreads) s_rgba[i] = __ldg(p.rgba + i);
    }
    if (RUBIX || SHARED_TABLE) __syncthreads();
}

// face byte b through plate `plate`'s tint LUT (stage_tables' copy)
__device__ __forceinline__ uint32_t tint(const uint32_t *s_lut, uint32_t plate, uint32_t b) { return reinterpret_cast<const uint8_t *>(s_lut)[plate * 256 + b]; }

// M_f, row-major, into M (left as it is without matrices: the rays are used as they are)
__device__ __forceinline__ void frame_matrix(const RayWarpParams &p, int f, float M[9]) {
    if (!p.xforms) return;
    const float *m = p.xforms + static_cast<size_t>(f) * p.xform_floats;
#pragma unroll
    for (int i = 0; i < 9; ++i) M[i] = __ldg(m + i);
}

// field pixel `at` of a frame's field, turned by M (as it is without matrices)
__device__ __forceinline__ void field_ray(const RayWarpParams &p, const float *field, size_t at, const float M[9], float t[3]) {
    const float *r = field + 3 * at;
    const float ray[3] = {__ldg(r), __ldg(r + 1), __ldg(r + 2)};
    t[0] = ray[0], t[1] = ray[1], t[2] = ray[2];
    if (p.xforms) turn_ray(M, ray, t);
}

// texel (x, y) of plate `plate` of a frame's faces: dense faces are the layout with rowbytes = ps
__device__ __forceinline__ const uint8_t *texel_at(const uint8_t *faces, const FaceLayoutParams &lay, uint32_t plate, uint32_t x, uint32_t y) {
    return faces + lay.plate_base[plate] + static_cast<size_t>(y) * lay.rowbytes + x;
}

// A frame's colour of a face byte b of plate `plate`: through the plate's tint LUT when RUBIX and the texel is off the
// rubix grid, then the frame's table (TABLES) or the shared one.  A background byte takes no tint.
template <bool RUBIX, bool TABLES>
struct FrameColours {
    const uint32_t *s_lut, *s_rgba, *table;

    __device__ __forceinline__ uint32_t operator()(uint32_t b, uint32_t plate = 0, bool on_grid = true) const {
        if (RUBIX && !on_grid) b = tint(s_lut, plate, b);
        return TABLES ? __ldg(table + b) : s_rgba[b];
    }
};

// f_rubix's grid tests of columns x0, x1 (bits 0, 1) and rows y0, y1 (bits 2, 3), as tap_colours takes them
__device__ __forceinline__ uint32_t grid_bits(const LensBuildParams &P, int x0, int x1, int y0, int y1) {
    return static_cast<uint32_t>(ray_on_rubix_line(P, x0)) | static_cast<uint32_t>(ray_on_rubix_line(P, x1)) << 1 |
           static_cast<uint32_t>(ray_on_rubix_line(P, y0)) << 2 | static_cast<uint32_t>(ray_on_rubix_line(P, y1)) << 3;
}

// The colours c[q] of the taps q = 00, 10, 01, 11 at columns x0 | x1 and rows y0 | y1 of plate `plate`, a tap being on
// the grid when its column or row is (grid: grid_bits)
template <bool RUBIX, bool TABLES>
__device__ __forceinline__ void tap_colours(const FrameColours<RUBIX, TABLES> &colour, const uint8_t *faces, const FaceLayoutParams &lay, uint32_t plate,
                                            uint32_t x0, uint32_t x1, uint32_t y0, uint32_t y1, uint32_t grid, uint32_t c[4]) {
    const uint8_t *row0 = texel_at(faces, lay, plate, 0, y0), *row1 = texel_at(faces, lay, plate, 0, y1);
    const uint32_t b[4] = {ld_texel(row0 + x0), ld_texel(row0 + x1), ld_texel(row1 + x0), ld_texel(row1 + x1)};
#pragma unroll
    for (int q = 0; q < 4; ++q) c[q] = colour(b[q], plate, ((grid >> (q & 1)) | (grid >> (2 + (q >> 1)))) & 1u);
}

// the blend of the four tap colours 00, 10, 01, 11 with 8-bit weights: the horizontal step in 16-bit lanes (255 * 256
// fits), the vertical one per byte in 32 bits
__device__ __forceinline__ uint32_t blend4(const uint32_t cq[4], uint32_t wx, uint32_t wy) {
    const uint32_t top_lo = (cq[0] & 0x00ff00ffu) * (256 - wx) + (cq[1] & 0x00ff00ffu) * wx;
    const uint32_t top_hi = ((cq[0] >> 8) & 0x00ff00ffu) * (256 - wx) + ((cq[1] >> 8) & 0x00ff00ffu) * wx;
    const uint32_t bot_lo = (cq[2] & 0x00ff00ffu) * (256 - wx) + (cq[3] & 0x00ff00ffu) * wx;
    const uint32_t bot_hi = ((cq[2] >> 8) & 0x00ff00ffu) * (256 - wx) + ((cq[3] >> 8) & 0x00ff00ffu) * wx;
    const auto blend = [wy](uint32_t t, uint32_t b) { return (t * (256 - wy) + b * wy + 32768u) >> 16; };
    return blend(top_lo & 0xffffu, bot_lo & 0xffffu) | blend(top_hi & 0xffffu, bot_hi & 0xffffu) << 8 | blend(top_lo >> 16, bot_lo >> 16) << 16 |
           blend(top_hi >> 16, bot_hi >> 16) << 24;
}

// The per-byte round-half-up mean (sum + S / 2) / S of S colours, summed in two SWAR words: bytes 0 and 2, bytes 1
// and 3, in 16-bit lanes (16 * 255 fits)
template <int S>
struct ColourMean {
    uint32_t lo = 0, hi = 0;

    __device__ __forceinline__ void add(uint32_t c) {
        if (S == 1) {
            lo = c;
            return;
        }
        lo += c & 0x00ff00ffu;
        hi += (c >> 8) & 0x00ff00ffu;
    }
    __device__ __forceinline__ uint32_t mean() const {
        if (S == 1) return lo;
        constexpr uint32_t half = S / 2;
        return ((lo & 0xffffu) + half) / S | (((hi & 0xffffu) + half) / S) << 8 | (((lo >> 16) + half) / S) << 16 | (((hi >> 16) + half) / S) << 24;
    }
};

// --------------------------------------------------------------------------
// One thread per item: a 4-pixel quad of a row (QUAD, W % 4 == 0) or one pixel.  The thread carries frames
// [blockIdx.y * frames_per_thread, ...): with one shared field it reads its rays once, and with one shared matrix too
// it maps them once; per frame it gathers the texels, tints, expands and stores like warp_gather_kernel (K1) /
// warp_scalar_kernel (K0).
// --------------------------------------------------------------------------
template <bool QUAD, bool RUBIX, bool RGBA, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads) ray_warp_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ LensBuildParams P,
                                                               const __grid_constant__ FaceLayoutParams lay) {
    constexpr int NP = QUAD ? 4 : 1;
    __shared__ uint32_t s_lut[RUBIX ? 6 * 256 / 4 : 1];
    __shared__ uint32_t s_rgba[RGBA && !TABLES ? 256 : 1];
    stage_tables<RUBIX, RGBA && !TABLES>(p, s_lut, s_rgba);

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
            frame_matrix(p, f, M);
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
                b = ld_texel(texel_at(faces, lay, plate, tx[k] & 0x1fffu, (tx[k] >> 13) & 0x1fffu));
                if (RUBIX && !(tx[k] & kOnGrid)) b = tint(s_lut, plate, b);
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
// Supersampled (ray_supersample_kernel) and bilinear (ray_bilinear_kernel, BILINEAR) RGBA: one thread per output pixel,
// whose K x K samples are the field pixels (K x + i, K y + j) of a dense K W x K H field, each turned and mapped as
// ray_warp_kernel maps a pixel's ray.  Sample j's row is 12 K contiguous bytes of the field, so a warp reads 384 K
// contiguous bytes per sub-row.  A mapped sample's colour is its texel's, or with BILINEAR the blend of its four taps'
// (x0 | x0 + 1, y0 | y0 + 1, clamped to its own plate) with the weights of ray_bilinear; an unmapped one is the pixel's
// background colour; the pixel is the ColourMean of the K^2 colours.  With one field and one matrix for every frame of
// the thread the packed samples are mapped once and carried; otherwise each frame re-reads its rays (a shared field of
// a small view from the caches; at 4K from HBM, which the per-sample arithmetic outweighs).
// (The minimum of one block per SM lets ptxas size the registers to the instance: with the default it held K = 2 with
// f_rubix to 64 registers and spilled.)
// --------------------------------------------------------------------------
template <bool BILINEAR, int K, bool RUBIX, bool KEEP, bool TABLES>
__device__ __forceinline__ void ray_samples(const RayWarpParams &p, const LensBuildParams &P, const FaceLayoutParams &lay) {
    constexpr int S = K * K;
    __shared__ uint32_t s_lut[RUBIX ? 6 * 256 / 4 : 1];
    __shared__ uint32_t s_rgba[TABLES ? 1 : 256];
    stage_tables<RUBIX, !TABLES>(p, s_lut, s_rgba);

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

    // a sample, packed in two words.  pos: its texel, or with BILINEAR its clamped first tap, x (bits 0-12) and y
    // (13-25), the plate (26-28), the second tap's steps dx (29) and dy (30) — 0 where the clamp folds both taps onto
    // one texel, and without BILINEAR — and mapped (31).  wt: wx (bits 0-7), wy (8-15), and with f_rubix grid_bits of
    // the taps' columns and rows (16-19; without BILINEAR, bit 16: the texel is on the grid).
    constexpr uint32_t kMapped = 0x80000000u;
    uint32_t pos[S], wt[S];
    int mapped = 0;
    for (int f = f0; f < f1; ++f) {
        if (f == f0 || !carry) {
            float M[9] = {};
            frame_matrix(p, f, M);
            const float *field = p.rays + static_cast<size_t>(f) * p.ray_floats;
            mapped = 0;
#pragma unroll
            for (int j = 0; j < K; ++j) {
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    float t[3];
                    field_ray(p, field, first + j * fw + i, M, t);
                    int plate = 0, x0 = 0, y0 = 0, wx = 0, wy = 0;
                    pos[j * K + i] = 0;
                    wt[j * K + i] = 0;
                    if (BILINEAR ? ray_bilinear(P, t, &plate, &x0, &y0, &wx, &wy) : ray_texel(P, t, &plate, &x0, &y0)) {
                        ++mapped;
                        const uint32_t tx = max(x0, 0), ty = max(y0, 0);
                        const uint32_t dx = BILINEAR && x0 >= 0 && x0 < ps - 1, dy = BILINEAR && y0 >= 0 && y0 < ps - 1;
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
                    wt[s] |= (BILINEAR ? grid_bits(P, tx, tx + dx, ty, ty + dy) : static_cast<uint32_t>(ray_on_rubix_grid(P, tx, ty))) << 16;
                }
            }
        }
        if (KEEP && mapped == 0) continue;
        const uint8_t *faces = p.faces + static_cast<size_t>(f) * p.face_stride;
        const FrameColours<RUBIX, TABLES> colour{s_lut, s_rgba, TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr};
        const uint32_t bgb = mapped < S ? __ldg(p.bg + pix) : 0u;
        ColourMean<S> sum;
#pragma unroll
        for (int s = 0; s < S; ++s) {
            uint32_t c;
            if (pos[s] & kMapped) {
                const uint32_t plate = (pos[s] >> 26) & 7u, x0 = pos[s] & 0x1fffu, y0 = (pos[s] >> 13) & 0x1fffu, grid = (wt[s] >> 16) & 0xfu;
                if (BILINEAR) {
                    uint32_t cq[4];
                    tap_colours(colour, faces, lay, plate, x0, x0 + ((pos[s] >> 29) & 1u), y0, y0 + ((pos[s] >> 30) & 1u), grid, cq);
                    c = blend4(cq, wt[s] & 0xffu, (wt[s] >> 8) & 0xffu);
                } else {
                    c = colour(ld_texel(texel_at(faces, lay, plate, x0, y0)), plate, grid & 1u);
                }
            } else {
                c = colour(bgb);
            }
            sum.add(c);
        }
        st_cs_u32(p.out + static_cast<size_t>(f) * p.out_stride + out_at, sum.mean());
    }
}

template <int K, bool RUBIX, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads, 1) ray_supersample_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ LensBuildParams P,
                                                                      const __grid_constant__ FaceLayoutParams lay) {
    ray_samples<false, K, RUBIX, KEEP, TABLES>(p, P, lay);
}

template <int K, bool RUBIX, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads, 1) ray_bilinear_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ LensBuildParams P,
                                                                   const __grid_constant__ FaceLayoutParams lay) {
    ray_samples<true, K, RUBIX, KEEP, TABLES>(p, P, lay);
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
// (min(2x + i, ps - 1), min(2y + j, ps - 1)), each the colour the nearest RGBA warp draws for that texel.
template <bool RUBIX, bool TABLES>
__global__ void __launch_bounds__(kRayThreads) ray_pyramid_base_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ RayPyramidParams q,
                                                                       const __grid_constant__ LensBuildParams P, const __grid_constant__ FaceLayoutParams lay) {
    __shared__ uint32_t s_lut[RUBIX ? 6 * 256 / 4 : 1];
    __shared__ uint32_t s_rgba[TABLES ? 1 : 256];
    stage_tables<RUBIX, !TABLES>(p, s_lut, s_rgba);
    const uint32_t s = q.size[1], ps = q.size[0];
    const uint32_t t = blockIdx.x * kRayThreads + threadIdx.x;
    if (t >= s * s) return;
    const uint32_t y = t / s, x = t - y * s, plate = blockIdx.y, f = blockIdx.z;
    const FrameColours<RUBIX, TABLES> colour{s_lut, s_rgba, TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr};
    const uint32_t x0 = 2 * x, x1 = min(2 * x + 1, ps - 1), y0 = 2 * y, y1 = min(2 * y + 1, ps - 1);
    uint32_t c[4];
    tap_colours(colour, p.faces + static_cast<size_t>(f) * p.face_stride, lay, plate, x0, x1, y0, y1, RUBIX ? grid_bits(P, x0, x1, y0, y1) : 0u, c);
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
// sample; its footprint is ray_footprint2 over the turned rays of its field neighbours, and ray_level gives L and w.
// Level 0's colour is ray_bilinear_kernel's at K = 1; level L >= 1's is the same blend on the pyramid's grid; the
// output mixes C_L and C_L+1 by w.  With one field and one matrix for every frame of the thread, the plate, (u, v), L,
// w and the level-0 grid tests are carried.
template <bool RUBIX, bool KEEP, bool TABLES>
__global__ void __launch_bounds__(kRayThreads, 1) ray_trilinear_kernel(const __grid_constant__ RayWarpParams p, const __grid_constant__ RayPyramidParams q,
                                                                    const __grid_constant__ LensBuildParams P, const __grid_constant__ FaceLayoutParams lay) {
    __shared__ uint32_t s_lut[RUBIX ? 6 * 256 / 4 : 1];
    __shared__ uint32_t s_rgba[TABLES ? 1 : 256];
    stage_tables<RUBIX, !TABLES>(p, s_lut, s_rgba);

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
    uint32_t grid = 0;   // f_rubix, level 0: grid_bits of the taps' columns and rows
    for (int f = f0; f < f1; ++f) {
        if (f == f0 || !carry) {
            float M[9] = {};
            frame_matrix(p, f, M);
            const float *field = p.rays + static_cast<size_t>(f) * p.ray_floats;
            float n[3];
            field_ray(p, field, pix, M, n);
            int px, py;
            mapped = ray_texel_uv(P, n, &plate, &px, &py, &u, &v);
            L = 0;
            w = 0;
            if (mapped) {
                // neighbour k of ray_footprint2, turned and normalised: (x + 1, y), (x - 1, y), (x, y + 1), (x, y - 1)
                const auto neighbour = [&](int k, float t[3]) {
                    if (!(k == 0 ? x + 1 < p.width : k == 1 ? x > 0 : k == 2 ? y + 1 < height : y > 0)) return false;
                    field_ray(p, field, k == 0 ? pix + 1 : k == 1 ? pix - 1 : k == 2 ? pix + p.width : pix - p.width, M, t);
                    ray_normalize3(t);
                    return true;
                };
                ray_level(ray_footprint2(P, plate, n, neighbour), q.lmax, &L, &w);
                if (RUBIX && L == 0) {
                    int x0, y0, wx, wy;
                    ray_bilinear_level(u, v, ps, &x0, &y0, &wx, &wy);
                    grid = grid_bits(P, max(x0, 0), min(x0 + 1, ps - 1), max(y0, 0), min(y0 + 1, ps - 1));
                }
            }
        }
        if (KEEP && !mapped) continue;
        const FrameColours<RUBIX, TABLES> colour{s_lut, s_rgba, TABLES ? p.rgba + static_cast<size_t>(f) * p.table_words : nullptr};
        uint32_t c;
        if (mapped) {
            const uint8_t *pyr = q.scratch + static_cast<size_t>(f) * q.stride;
            if (L == 0) {
                int x0, y0, wx, wy;
                ray_bilinear_level(u, v, ps, &x0, &y0, &wx, &wy);
                uint32_t cq[4];
                tap_colours(colour, p.faces + static_cast<size_t>(f) * p.face_stride, lay, plate, max(x0, 0), min(x0 + 1, ps - 1), max(y0, 0),
                            min(y0 + 1, ps - 1), grid, cq);
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
            c = colour(__ldg(p.bg + pix));
        }
        st_cs_u32(p.out + static_cast<size_t>(f) * p.out_stride + out_at, c);
    }
}

// ---- dispatch ---------------------------------------------------------------------------------------------------------

// f(std::true_type{}) or f(std::false_type{}): a runtime flag as a compile-time constant
template <class F>
void with_flag(bool on, F &&f) {
    if (on) f(std::true_type{});
    else f(std::false_type{});
}

// f(std::integral_constant<int, K>{}) for the first K of the list equal to k, else for the last
template <int K, int... Ks, class F>
void with_factor(int k, F &&f) {
    if constexpr (sizeof...(Ks) == 0) f(std::integral_constant<int, K>{});
    else if (k == K) f(std::integral_constant<int, K>{});
    else with_factor<Ks...>(k, f);
}

RayPyramidParams pyramid_params(const RayWarpLaunch &L) {
    RayPyramidParams q;
    memset(&q, 0, sizeof q);
    q.scratch = static_cast<uint8_t *>(L.q.scratch);
    q.stride = L.c.pyramid_bytes;
    q.lmax = L.c.lmax;
    for (int l = 0; l <= L.c.lmax; ++l) {
        q.size[l] = static_cast<uint32_t>(L.c.level_size[l]);
        q.off[l] = L.c.level_off[l];
    }
    return q;
}

// the pyramid of every frame: one launch per level 1..lmax, the base instance of (rubix, tables) first
void launch_pyramids(const RayWarpLaunch &L, const RayWarpParams &p, const RayPyramidParams &q, cudaStream_t st) {
    for (int l = 1; l <= L.c.lmax; ++l) {
        const uint32_t s = q.size[l];
        const dim3 g((s * s + kRayThreads - 1) / kRayThreads, static_cast<unsigned>(L.globe.numplates), static_cast<unsigned>(L.r.nframes));
        if (l > 1) ray_pyramid_reduce_kernel<<<g, kRayThreads, 0, st>>>(q, l);
        else
            with_flag(L.rubix, [&](auto rubix) {
                with_flag(L.tables(), [&](auto tables) { ray_pyramid_base_kernel<rubix, tables><<<g, kRayThreads, 0, st>>>(p, q, L.globe, L.c.layout); });
            });
    }
}

}  // namespace

bool launch_ray_warp(const RayWarpLaunch &L, std::string *name, int *cuda_err) {
    RayWarpParams p;
    p.rays = L.q.rays;
    p.ray_floats = L.q.ray_stride / 4;
    p.xforms = L.q.xforms;
    p.xform_floats = L.q.xform_stride / 4;
    p.faces = static_cast<const uint8_t *>(L.r.faces);
    p.face_stride = L.r.face_stride;
    p.bg = L.bg;
    p.lut = L.lut;
    p.rgba = L.palette;
    p.table_words = L.r.table_stride / 4;
    p.out = L.c.view;
    p.out_stride = L.r.out_stride;
    p.pitch = static_cast<uint32_t>(L.c.pitch);
    p.width = static_cast<uint32_t>(L.width);
    p.nitems = L.shape.nitems;
    p.nframes = L.r.nframes;
    p.frames_per_thread = L.shape.frames_per_thread;
    const dim3 grid(L.shape.grid_x, L.shape.grid_y);
    cudaStream_t st = static_cast<cudaStream_t>(L.r.stream);
    const bool trilinear = L.q.filter == RayFilter::Trilinear;
    const int factor = L.q.factor;
    const bool keep = L.r.keep_unmapped, tables = L.tables();
    const RayPyramidParams q = pyramid_params(L);
    if (trilinear) launch_pyramids(L, p, q, st);
    // instances: per-frame tables exist only in RGBA (ray_warp_kernel: 24), supersampled K = 2..4 (24), bilinear
    // K = 1..4 (32), trilinear (8)
    with_flag(L.rubix, [&](auto rubix) {
        with_flag(keep, [&](auto keep) {
            with_flag(tables, [&](auto tables) {
                if (trilinear) {
                    ray_trilinear_kernel<rubix, keep, tables><<<grid, kRayThreads, 0, st>>>(p, q, L.globe, L.c.layout);
                } else if (L.q.filter == RayFilter::Bilinear) {
                    with_factor<1, 2, 3, 4>(factor, [&](auto k) { ray_bilinear_kernel<k, rubix, keep, tables><<<grid, kRayThreads, 0, st>>>(p, L.globe, L.c.layout); });
                } else if (factor > 1) {
                    with_factor<2, 3, 4>(factor, [&](auto k) { ray_supersample_kernel<k, rubix, keep, tables><<<grid, kRayThreads, 0, st>>>(p, L.globe, L.c.layout); });
                } else {
                    with_flag(L.shape.quads, [&](auto quad) {
                        with_flag(L.r.rgba, [&](auto rgba) {
                            ray_warp_kernel<quad, rubix, rgba, keep, rgba && tables><<<grid, kRayThreads, 0, st>>>(p, L.globe, L.c.layout);
                        });
                    });
                }
            });
        });
    });
    char args[64], buf[192];
    if (trilinear) snprintf(args, sizeof args, "rubix=%d,keep=%d,tables=%d", L.rubix, keep, tables);
    else if (L.q.filter == RayFilter::Bilinear || factor > 1) snprintf(args, sizeof args, "k=%d,rubix=%d,keep=%d,tables=%d", factor, L.rubix, keep, tables);
    else snprintf(args, sizeof args, "quad=%d,rubix=%d,rgba=%d,keep=%d,tables=%d", L.shape.quads, L.rubix, L.r.rgba, keep, tables);
    const int n = snprintf(buf, sizeof buf, "%s<%s> grid=(%u,%u) block=%d frames/thread=%d", ray_warp_kernel_name(L.q.filter, factor), args, grid.x, grid.y,
                           kRayThreads, L.shape.frames_per_thread);
    if (trilinear) snprintf(buf + n, sizeof buf - n, " levels=%d", L.c.lmax);
    *name = buf;
    const cudaError_t e = cudaGetLastError();
    *cuda_err = static_cast<int>(e);
    return e == cudaSuccess;
}

}  // namespace blinky
