// Device side of the H100 lens-warp path: resident lensmap / LUTs, the warp
// kernels and the host<->device frame pipeline.  CUDA types are kept out of
// this header so that plain C++ translation units can include it.
//
// Replaces the reference's per-frame hot loop, render_lensmap()
// (the reference's engine/NQ/fisheye.c:2406-2424).
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace blinky {

struct TilePlan;  // tile_plan.h

struct LensmapUpload {
    int width = 0, height = 0, platesize = 0, numplates = 0;
    const uint32_t *packed = nullptr;        // [height*width]
    const uint8_t *palmaps = nullptr;        // [6*256]
    int display[6] = {0, 0, 0, 0, 0, 0};
    int plate_rect[6][4] = {};               // texel rectangle each plate is sampled in (x0,y0,x1,y1)
    bool rubix = false;
    const int32_t *span_off = nullptr;       // [height+1]
    const int32_t *spans = nullptr;          // pairs
    size_t nspans = 0;
    const TilePlan *plan = nullptr;          // tiled layout (may be null: flat kernels only)
};

class WarpDevice {
public:
    // throws std::runtime_error on CUDA failure
    explicit WarpDevice(int device);
    ~WarpDevice();

    int device() const { return device_; }
    const std::string &last_error() const { return err_; }

    bool upload_lensmap(const LensmapUpload &lm);
    void set_rubix(bool on) { rubix_ = on; }
    bool set_background(const uint8_t *bg_host);   // [H][W] or nullptr -> zeros
    bool set_rgba_table(const uint32_t table[256]);
    void set_kernel(int variant) { variant_ = variant; }

    // device-resident batch (asynchronous on `stream`, nullptr = CUDA default stream)
    bool warp(const void *d_faces, size_t face_stride, void *d_out, size_t out_stride, int nframes, void *stream,
              bool rgba);
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
    size_t upload_bytes_per_frame() const;
    const std::string &last_kernel() const { return last_kernel_; }

private:
    struct Slot;
    bool ensure_slots();
    bool fail(const char *what, int cuda_err);
    void finalize_slot(Slot &s);

    int device_ = 0;
    int sm_count_ = 132;
    void *stream_ = nullptr;  // cudaStream_t
    bool upload_by_kernel_ = false, out_by_kernel_ = false;  // warp_host variants (BLINKY_E2E_UPLOAD / BLINKY_E2E_OUT)
    bool batch_copies_ = true;   // plate rectangles of a frame in one cudaMemcpy3DBatchAsync (BLINKY_E2E_BATCH=0: one 2-D copy each)
    const void *pin_src_ptr_ = nullptr, *pin_dst_ptr_ = nullptr;  // last buffers warp_host saw and whether they are pinned
    bool pin_src_ = false, pin_dst_ = false;
    std::string err_;

    // resident lensmap
    int width_ = 0, height_ = 0, platesize_ = 0, numplates_ = 0;
    size_t npix_ = 0, npix_pad_ = 0;
    int display_[6] = {0, 0, 0, 0, 0, 0};
    int plate_rect_[6][4] = {};
    bool rubix_ = false;
    bool have_lensmap_ = false;
    uint32_t *d_lensmap_ = nullptr;
    uint8_t *d_lut_ = nullptr;
    uint8_t *d_bg_ = nullptr;
    uint32_t *d_rgba_ = nullptr;
    bool have_rgba_ = false;
    std::vector<int32_t> span_off_, spans_;
    int variant_ = 0;

    // tiled layout (ring kernel)
    struct TmapSet;
    struct TicketCounter {
        void *stream = nullptr;
        uint32_t *d_counter = nullptr;
        uint32_t base = 0;  // value the counter will have when the next launch on this stream starts
    };
    bool have_plan_ = false;
    bool plan_has_box_ = false;
    void *d_tiles_ = nullptr;       // TileDesc[]
    uint8_t *d_entries_ = nullptr;
    uint32_t ntiles_ = 0, nbox_tiles_ = 0, ngather_tiles_ = 0;
    int stage_bytes_ = 0;                // largest staged box of the plan
    int static_pct_ = 85;                // share of the ring kernel's units scheduled statically (BLINKY_STATIC_PCT)
    int l2_promotion_ = 0;               // CUtensorMapL2promotion of the box descriptors (BLINKY_L2_PROMOTION)
    bool serial_gather_ = false;         // BLINKY_SERIAL_GATHER=1: GATHER tiles in their own kernel instead of as extra CTAs of the ring kernel's launch
    int ring_bytes_override_ = 0, ring_ctas_cap_ = 0, fchunk_ = 0;  // tuning overrides (BLINKY_RING_BYTES / _CTAS, BLINKY_FCHUNK); 0 = automatic
    int merged_items_max_ = 4096;        // gather items up to which GATHER tiles ride in the ring kernel's launch whatever their share (BLINKY_MERGED_ITEMS)
    int ring_boxes_ = 0;                 // boxes a warp keeps in flight at most (BLINKY_RING_BOXES)
    size_t smem_per_sm_ = 233472;
    std::vector<uint16_t> shapes_;
    std::vector<TmapSet *> tmap_sets_;   // small cache keyed by (faces ptr, stride, nframes)
    uint64_t tmap_tick_ = 0;
    std::vector<TicketCounter> tickets_; // one work counter per stream the ring kernel was launched on
    void *encode_fn_ = nullptr;          // cuTensorMapEncodeTiled
    int ring_ctas_per_sm_[4] = {0, 0, 0, 0};
    size_t ring_smem_[4] = {0, 0, 0, 0};
    TmapSet *get_tmaps(const void *d_faces, size_t face_stride, int nframes);
    bool launch_ring(const void *d_faces, size_t face_stride, void *d_out, size_t out_stride, int nframes, void *stream,
                     bool rgba);
    bool launch_flat(const void *d_faces, size_t face_stride, void *d_out, size_t out_stride, int nframes, void *stream,
                     bool rgba);
    std::string plan_summary_;
public:
    const std::string &plan_summary() const { return plan_summary_; }
private:

    // e2e pipeline
    std::vector<Slot *> slots_;
    size_t slot_face_bytes_ = 0, slot_out_bytes_ = 0;
    static constexpr int kMaxHostGroup = 8;
    int host_group_ = 1;                 // frames per slot of the blinky_warp_host pipeline (BLINKY_HOST_GROUP)

    int64_t launches_ = 0;
    std::string last_kernel_;
};

}  // namespace blinky
