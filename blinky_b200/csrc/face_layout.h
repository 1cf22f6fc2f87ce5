// Face layout (blinky_set_face_layout): where the plates of a frame sit in the caller's surface.
//
// A layout is one row pitch `rowbytes` and an origin (x_i, y_i) per plate, in bytes and rows.  Texel
// (px, py) of plate i lies at  frame + (y_i + py) * rowbytes + x_i + px.  The lensmap and the tile plan
// keep addressing texels in plate space (plate * ps^2 + py * ps + px); the kernels split such an offset
// with layout_texel() below.  Host and device share this header, so the CPU tests can pin the split.
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define BLINKY_HD __host__ __device__ __forceinline__
#else
#define BLINKY_HD inline
#endif

namespace blinky {

// n / d as ((umulhi(n, mul) + n) >> shift), exact for every n < 2^28 (the lensmap's texel index):
// with s = ceil(log2 d) and m = ceil(2^(32+s) / d) = mul + 2^32, the error of n * m / 2^(32+s) against
// n / d is n * (m * d - 2^(32+s)) / (d * 2^(32+s)) < n / 2^(32+s) < 2^-4 / 2^s < 1 / d (as d <= 2^s),
// too small to carry the quotient past the next integer.
struct FastDiv {
    uint32_t mul, shift;
};

inline FastDiv make_fastdiv(uint32_t d) {   // 1 <= d <= 2^28
    uint32_t s = 0;
    while ((uint64_t{1} << s) < d) ++s;
    const uint64_t m = ((uint64_t{1} << (32 + s)) + d - 1) / d;
    return {static_cast<uint32_t>(m - (uint64_t{1} << 32)), s};
}

BLINKY_HD uint32_t fastdiv(uint32_t n, FastDiv d) {
#if defined(__CUDA_ARCH__)
    const uint32_t hi = __umulhi(n, d.mul);
#else
    const uint32_t hi = static_cast<uint32_t>((static_cast<uint64_t>(n) * d.mul) >> 32);
#endif
    return (hi + n) >> d.shift;   // (n < 2^28: no overflow)
}

constexpr int kLayoutPlates = 6;

// The layout as the kernels read it: their last parameter (the dense instances never read it).
struct FaceLayoutParams {
    uint64_t plate_base[kLayoutPlates];   // byte offset of texel (0, 0) of plate i in a frame: y_i * rowbytes + x_i
    int32_t org_x[kLayoutPlates], org_y[kLayoutPlates];   // the plate's origin: shifts a TMA box from plate to surface coordinates
    uint32_t rowbytes;
    uint32_t ps, ps2;                     // plate size, plate size squared
    FastDiv div_ps2, div_ps;
};

// byte offset in a frame's surface of the texel at plate-space offset `off` (< 2^28, of a plate < 6)
BLINKY_HD size_t layout_texel(uint32_t off, const FaceLayoutParams &L) {
    const uint32_t plate = fastdiv(off, L.div_ps2);
    const uint32_t rem = off - plate * L.ps2;
    const uint32_t py = fastdiv(rem, L.div_ps);
    const uint32_t px = rem - py * L.ps;
    return static_cast<size_t>(L.plate_base[plate]) + static_cast<size_t>(py) * L.rowbytes + px;
}

}  // namespace blinky
