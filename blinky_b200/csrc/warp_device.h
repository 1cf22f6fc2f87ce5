// Device side of the H100 lens-warp path: resident lensmap / LUTs, the warp
// kernels and the host<->device frame pipeline.  CUDA types are kept out of
// this header so that plain C++ translation units can include it.
//
// Replaces the reference's per-frame hot loop, render_lensmap()
// (the reference's engine/NQ/fisheye.c:2406-2424).
#pragma once

#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "device_buffer.h"
#include "face_layout.h"
#include "ray_texel.h"   // kRayMaxLevels

namespace blinky {

struct DevicePlan;     // tile_plan_device.h
struct KernelVariant;  // launch_plan.h
enum class WarpKernel;

// What WarpDevice::install keeps of a lensmap beside its device buffers (DevicePlan).
struct LensmapUpload {
    int width = 0, height = 0, platesize = 0, numplates = 0;
    const uint8_t *palmaps = nullptr;        // [6*256]
    int display[6] = {0, 0, 0, 0, 0, 0};
    int plate_rect[6][4] = {};               // texel rectangle each plate is sampled in (x0,y0,x1,y1)
    bool rubix = false;
    const int32_t *span_off = nullptr;       // [height+1]
    const int32_t *spans = nullptr;          // pairs
    size_t nspans = 0;
};

// The entry point a warp request comes from (warp_entry_name): it decides which checks the request gets, in which
// order, and how its refusals read (check_warp, launch_plan.h).
enum class WarpEntry {
    Internal,                                 // blinky_warp_host's frames and the sharded batches
    Dense, DenseRgba,                         // blinky_warp_device[_rgba]: the view is the whole of out
    View, ViewRgba, ViewRgbaTables,           // blinky_warp_device_view*: the view rectangle at (x0, y0) of out
    Rays, RaysRgba, RaysSupersampled, RaysBilinear, RaysTrilinear,   // blinky_warp_device_rays*: likewise
    PyramidBytes,                             // blinky_ray_pyramid_bytes: the ray warps' checks of the state alone
    Host,                                     // blinky_warp_host: the view rectangle at (x0, y0) of a host buffer
};

// One device-resident batch (WarpDevice::warp), asynchronous on `stream` (nullptr = CUDA's default stream).  May be
// captured into a CUDA graph: see WarpDevice::release_captures.
struct WarpRequest {
    WarpRequest(const void *faces, size_t face_stride, void *out, size_t out_stride, int nframes, void *stream)
        : faces(faces), face_stride(face_stride), out(out), out_stride(out_stride), nframes(nframes), stream(stream) {}
    const void *faces;                 // frame 0's faces, in the face layout (WarpDevice::set_face_layout)
    size_t face_stride;                // bytes between frames
    void *out;                         // frame 0's screen, whose view rectangle at (x0, y0) the warp writes
    size_t out_stride;                 // bytes between frames
    int nframes;
    void *stream;                      // cudaStream_t
    WarpEntry entry = WarpEntry::Internal;
    int rowbytes = 0, x0 = 0, y0 = 0;  // the screen's bytes between rows and the view's origin in it (view entry points
                                       // and Host; otherwise 0: the view is the whole screen, rows W * bytes per pixel apart)
    bool rgba = false;
    bool keep_unmapped = false;        // only mapped pixels are written, the others keep what the caller's buffer holds
    // RGBA: frame f is expanded through the 256-entry device table at tables + f * table_stride bytes (table_stride 0:
    // one table for every frame) instead of set_rgba_table's, read when the launch runs.  tables 16-byte aligned,
    // table_stride a multiple of 16.
    const uint32_t *tables = nullptr;
    size_t table_stride = 0;
    bool dense_faces = false;          // the faces are dense [plate][ps][ps] frames whatever the face layout

    // frame 0's view origin, in screens whose rows are `pitch` bytes apart
    uint8_t *view(size_t pitch) const { return static_cast<uint8_t *>(out) + static_cast<size_t>(y0) * pitch + static_cast<size_t>(x0) * (rgba ? 4 : 1); }
};

// How each sample of a ray warp takes its colour: the nearest texel (ray_warp_kernel at factor 1,
// ray_supersample_kernel at 2-4), four texels blended (ray_bilinear_kernel, factor 1-4), or two mip levels' bilinear
// colours blended (the pyramid launches, then ray_trilinear_kernel, factor 1).  Every filter but Nearest at factor 1
// writes RGBA.
enum class RayFilter { Nearest, Bilinear, Trilinear };

// The ray field and matrices of a warp from rays (WarpDevice::warp_rays), device memory read when the launch runs.
struct RayRequest {
    const float *rays = nullptr;   // frame 0's field, float32[height][width][3] as blinky_set_raymap reads it
    size_t ray_stride = 0;         // bytes between frames (0: one field for every frame)
    const float *xforms = nullptr; // frame 0's 3x3 matrix, row-major (nullptr: the rays as they are)
    size_t xform_stride = 0;       // bytes between frames (0: one matrix for every frame)
    int factor = 1;             // 2-4: a [factor * height][factor * width] field, factor^2 samples averaged per RGBA pixel
    RayFilter filter = RayFilter::Nearest;   // Bilinear: factor 1-4; Trilinear: factor 1, the two mip levels around the footprint
    void *scratch = nullptr;    // trilinear: the frames' pyramids, frame f at scratch + f * B (16-byte aligned)
    size_t scratch_bytes = 0;   // trilinear: at least nframes * B
};

// What the checks of a warp read besides the call (check_warp): the installed lensmap, the globe and the face layout.
struct GlobeState {
    bool valid = false;
    bool plate_script = false;         // the globe picks its plates with a globe_plate script
    int plates = 0;
};
struct WarpState {
    int width = 0, height = 0, platesize = 0;   // the installed view (0 before the first install)
    const int *display = nullptr;               // [6]: with plate_rect, the plates the lensmap samples
    const int (*plate_rect)[4] = nullptr;       // [6] texel rectangles (x0, y0, x1, y1)
    GlobeState globe;
    int layout_rowbytes = 0;                    // face layout: 0 = dense
    const int32_t *layout_origins = nullptr;    // (x, y) per plate
    int layout_plates = 0;
};

// What check_warp derives for an accepted call.
struct CheckedWarp {
    bool launch = false;         // false: nframes <= 0, nothing to do
    uint8_t *view = nullptr;     // frame 0's view origin, WarpRequest::view(pitch)
    size_t pitch = 0;            // bytes between the view's rows
    bool use_layout = false;     // the faces are read through `layout` (ray warps: always, dense faces included)
    FaceLayoutParams layout = {};
    uint32_t layout_rows = 0;    // rows of a frame's surface in the face layout
    // trilinear (and blinky_ray_pyramid_bytes): the frames' pyramids, ray_pyramid_levels
    int lmax = 0;
    int level_size[kRayMaxLevels] = {};
    uint64_t level_off[kRayMaxLevels] = {};
    uint64_t pyramid_bytes = 0;
};

class WarpDevice {
public:
    // throws std::runtime_error on CUDA failure
    explicit WarpDevice(int device);
    ~WarpDevice();

    int device() const { return device_; }
    const std::string &last_error() const { return err_; }

    // Makes lm, with plan's map and tile plan (whose buffers it takes over), the resident lensmap, and copies
    // lm.palmaps into the LUTs.  All or nothing: on failure the current lensmap stays resident.
    bool install(const LensmapUpload &lm, DevicePlan &&plan);
    // the plates' palette LUTs, rewritten in place (graphs captured earlier read them too)
    bool set_luts(const uint8_t palmaps[6 * 256]);
    void set_rubix(bool on) { rubix_ = on; }
    bool set_background(const uint8_t *bg_host);   // [H][W] or nullptr -> zeros
    bool set_rgba_table(const uint32_t table[256]);
    void set_kernel(int variant) { variant_ = variant; }
    // face layout (face_layout.h) of the faces every later warp reads: rowbytes 0 = dense [plate][ps][ps] frames;
    // origins: nplates (x, y) pairs.  Checked against the lensmap at each warp (BLINKY_E_INVALID when it does not fit).
    void set_face_layout(int rowbytes, const int32_t *origins, int nplates);

    // size of the resident lensmap's view (0 before the first install)
    int width() const;
    int height() const;
    int platesize() const;
    // entries of a device lensmap buffer for npix pixels (the kernels read whole blocks; the padding is unmapped)
    static size_t padded_pixels(size_t npix);
    // copies of the resident map ([height][width] entries) and tile plan, synchronously
    bool download_lensmap(uint32_t *out);
    bool download_plan(void *tiles, void *entries, size_t entry_bytes);
    size_t plan_tiles() const;
    size_t plan_entry_bytes() const;

    // what the checks of a warp read of this object, with the globe `globe`
    WarpState state(const GlobeState &globe = {}) const;
    // r, checked (check_warp) and launched: nothing is launched when it is refused
    bool warp(const WarpRequest &r);
    // r (view, rgba, keep_unmapped, tables) with each pixel's texel computed from its ray in q, turned, through the
    // globe `params` (FisheyeHost::device_params at the resident view's size) described by `globe`: the resident
    // lensmap gives only the view's size and background.  Every plate of the globe must have an origin in the face
    // layout.  Capturable like warp().  q.factor > 1: the supersampled RGBA warp (ray_supersample_kernel);
    // Bilinear: the bilinear RGBA warp at any factor (ray_bilinear_kernel); Trilinear: the frames' pyramids in
    // q.scratch, then the trilinear RGBA warp (ray_trilinear_kernel), lmax + 1 launches.
    bool warp_rays(const WarpRequest &r, const RayRequest &q, const GlobeState &globe, const LensBuildParams &params);
    // The caller will not run again any graph that captured a warp of this object: synchronises the device, lets go
    // of the generations held for such graphs and returns every capture counter slot to the pool.
    bool release_captures();
    // BLINKY_E_* code of the last failure (BLINKY_E_CUDA unless the call was refused for another reason)
    int last_error_code() const { return err_code_; }
    // end to end from host buffers (synchronous): r.faces and r.out in host memory, 8-bit, entry Host
    bool warp_host(const WarpRequest &r);

    bool alloc_device(size_t bytes, void **out);
    bool free_device(void *p);
    bool ipc_export(void *p, unsigned char handle[64]);
    bool ipc_open(const unsigned char handle[64], void **out);
    bool ipc_close(void *p);
    bool alloc_pinned(size_t bytes, void **out);
    bool free_pinned(void *p);
    bool sync();

    int64_t launches() const { return launches_; }
    const std::string &last_kernel() const { return last_kernel_; }

private:
    struct Generation;
    struct Slot;
    bool ensure_slots();
    bool fail(const char *what, int cuda_err);
    // check_warp of r (and q) on state(globe): false, with the refusal in err_code_ / err_, or the derived values in *c
    bool check(const WarpRequest &r, const RayRequest &q, const GlobeState &globe, CheckedWarp *c);
    // whether r.stream is capturing (and which capture); remember_capture: a warp was captured into it
    bool capture_info(void *stream, bool *capturing, unsigned long long *id);
    void remember_capture(void *stream, unsigned long long id);
    void finalize_slot(Slot &s);

    int device_ = 0;
    int sm_count_ = 132;
    int threads_per_sm_ = 2048;
    bool batch_copies_ = true;   // plate rectangles of a frame in one cudaMemcpy3DBatchAsync (false once the driver refused it)
    const void *pin_src_ptr_ = nullptr, *pin_dst_ptr_ = nullptr;  // last buffers warp_host saw and whether they are pinned
    bool pin_src_ = false, pin_dst_ = false;
    std::string err_;
    int err_code_ = 0;

    // the resident lensmap, its plan and background (null before the first install); warp() reads it through this
    // one pointer
    std::shared_ptr<const Generation> cur_;
    bool rubix_ = false;
    DeviceBuffer d_lut_;    // uint8_t[6][256]
    DeviceBuffer d_rgba_;   // uint32_t[256]
    int variant_ = 0;
    int layout_rowbytes_ = 0;              // face layout: 0 = dense
    std::vector<int32_t> layout_origins_;  // (x, y) per plate

    // tiled layout (ring kernel)
    struct TmapSet;
    struct TicketCounter {
        void *stream = nullptr;
        DeviceBuffer counter;  // uint32_t, 0 between launches: each launch sets it back
    };
    int static_pct_ = 85;                // share of the ring kernel's units scheduled statically (BLINKY_STATIC_PCT)
    bool serial_gather_ = false;         // BLINKY_SERIAL_GATHER=1: GATHER tiles in their own kernel instead of as extra CTAs of the ring kernel's launch
    int ring_bytes_override_ = 0, ring_ctas_cap_ = 0, fchunk_ = 0;  // tuning overrides (BLINKY_RING_BYTES / _CTAS, BLINKY_FCHUNK); 0 = automatic
    int merged_items_max_ = 4096;        // gather items up to which GATHER tiles ride in the ring kernel's launch of <= 8 frames (BLINKY_MERGED_ITEMS)
    int ring_boxes_ = 0;                 // boxes a warp keeps in flight at most (BLINKY_RING_BOXES)
    size_t smem_per_sm_ = 233472;
    std::vector<std::unique_ptr<TmapSet>> tmap_sets_;   // small cache keyed by (faces ptr, stride, nframes, face layout's surface)
    uint64_t tmap_tick_ = 0;
    std::vector<TicketCounter> tickets_; // one work counter per stream the ring kernel was launched on (eagerly)
    void *encode_fn_ = nullptr;          // cuTensorMapEncodeTiled
    int ring_ctas_per_sm_[32] = {};      // per ring kernel instance (KernelVariant::index)
    size_t ring_smem_[32] = {};
    TmapSet *get_tmaps(const void *d_faces, size_t face_stride, int nframes, uint32_t rowbytes, uint32_t rows);
    // r as check_warp accepted it, with what it derived in c
    bool launch_ring(const WarpRequest &r, const CheckedWarp &c, const KernelVariant &v, bool capturing);
    bool launch_flat(const WarpRequest &r, const CheckedWarp &c, const KernelVariant &v, WarpKernel k);

    // CUDA graph capture.  A captured ring launch gets a work counter of its own out of a pool allocated (zeroed) with
    // the object, because its graph may be replayed on any stream, beside eager launches and other graphs; slots are
    // handed out in order and come back all at once (release_captures).  The generations captured launches read stay
    // held, past the install that replaces them, until release_captures.
    struct CaptureStream {
        void *stream;
        unsigned long long id;  // capture sequence a warp was captured into
    };
    DeviceBuffer d_capture_slots_;        // uint32_t[kCaptureSlots]
    uint32_t capture_slots_used_ = 0;
    std::vector<std::shared_ptr<const Generation>> held_;  // generations captured graphs may read
    std::vector<CaptureStream> capture_streams_;  // where warps were captured (release_captures refuses while one is open)

    // e2e pipeline
    std::vector<std::unique_ptr<Slot>> slots_;
    size_t slot_face_bytes_ = 0, slot_out_bytes_ = 0;

    int64_t launches_ = 0;
    std::string last_kernel_;
};

}  // namespace blinky
