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
#include "ray_warp.h"   // RayFilter

namespace blinky {

struct DevicePlan;     // tile_plan_device.h
struct KernelVariant;  // launch_plan.h
struct LensBuildParams;  // lens_device.h
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

// One device-resident batch (WarpDevice::warp), asynchronous on `stream` (nullptr = CUDA's default stream).  May be
// captured into a CUDA graph: see WarpDevice::release_captures.
struct WarpRequest {
    WarpRequest(const void *faces, size_t face_stride, void *out, size_t out_stride, int nframes, void *stream)
        : faces(faces), face_stride(face_stride), out(out), out_stride(out_stride), nframes(nframes), stream(stream) {}
    const void *faces;                 // frame 0's faces, in the face layout (WarpDevice::set_face_layout)
    size_t face_stride;                // bytes between frames
    void *out;                         // view origin of frame 0
    size_t out_stride;                 // bytes between frames
    size_t out_pitch = 0;              // bytes between rows (0: dense, W * bytes per pixel)
    int nframes;
    void *stream;                      // cudaStream_t
    bool rgba = false;
    bool keep_unmapped = false;        // only mapped pixels are written, the others keep what the caller's buffer holds
    // RGBA: frame f is expanded through the 256-entry device table at tables + f * table_stride bytes (table_stride 0:
    // one table for every frame) instead of set_rgba_table's, read when the launch runs.  tables 16-byte aligned,
    // table_stride a multiple of 16.
    const uint32_t *tables = nullptr;
    size_t table_stride = 0;
    bool dense_faces = false;          // the faces are dense [plate][ps][ps] frames whatever the face layout
};

// The ray field and matrices of a warp from rays (WarpDevice::warp_rays), device memory read when the launch runs.
struct RayRequest {
    const float *rays;          // frame 0's field, float32[height][width][3] as blinky_set_raymap reads it
    size_t ray_stride;          // bytes between frames (0: one field for every frame)
    const float *xforms;        // frame 0's 3x3 matrix, row-major (nullptr: the rays as they are)
    size_t xform_stride;        // bytes between frames (0: one matrix for every frame)
    int factor = 1;             // 2-4: a [factor * height][factor * width] field, factor^2 samples averaged per RGBA pixel
    RayFilter filter = RayFilter::Nearest;   // Bilinear: factor 1-4; Trilinear: factor 1, the two mip levels around the footprint
    void *scratch = nullptr;    // trilinear: the frames' pyramids, frame f at scratch + f * B (16-byte aligned)
    size_t scratch_bytes = 0;   // trilinear: at least nframes * B
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

    bool warp(const WarpRequest &r);
    // r (view, rgba, keep_unmapped, tables) with each pixel's texel computed from its ray in q, turned, through the
    // globe `globe` (FisheyeHost::device_params at the resident view's size, no globe_plate script): the resident
    // lensmap gives only the view's size and background.  Every plate of the globe must have an origin in the face
    // layout.  Capturable like warp().  q.factor > 1: the supersampled RGBA warp (ray_supersample_kernel);
    // Bilinear: the bilinear RGBA warp at any factor (ray_bilinear_kernel); Trilinear: the frames' pyramids in
    // q.scratch, then the trilinear RGBA warp (ray_trilinear_kernel), lmax + 1 launches.
    bool warp_rays(const WarpRequest &r, const RayRequest &q, const LensBuildParams &globe);
    // The caller will not run again any graph that captured a warp of this object: synchronises the device, lets go
    // of the generations held for such graphs and returns every capture counter slot to the pool.
    bool release_captures();
    // BLINKY_E_* code of the last failure (BLINKY_E_CUDA unless the call was refused for another reason)
    int last_error_code() const { return err_code_; }
    // end to end from host buffers (synchronous)
    bool warp_host(const uint8_t *faces_host, size_t face_stride, uint8_t *dst_host, size_t dst_frame_stride,
                   int dst_rowbytes, int x0, int y0, int nframes, bool keep_unmapped);

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
    // globe_plates >= 0: the plates 0..globe_plates-1 need an origin (a warp from rays may sample any of them), instead
    // of the plates the lensmap samples
    bool make_layout(size_t face_stride, int nframes, FaceLayoutParams *lay, int globe_plates = -1);
    // the checks every warp makes of its output; *pitch: the bytes between output rows
    bool check_output(const WarpRequest &r, size_t *pitch);
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
    uint32_t layout_rows_ = 0;             // rows of a frame's surface (set by make_layout)

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
    // what warp() derived from the request: pitch, the output's bytes between rows; lay, the face layout when v.layout
    // (zero otherwise)
    bool launch_ring(const WarpRequest &r, uint32_t pitch, const KernelVariant &v, const FaceLayoutParams &lay, bool capturing);
    bool launch_flat(const WarpRequest &r, uint32_t pitch, const KernelVariant &v, const FaceLayoutParams &lay, WarpKernel k);

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
