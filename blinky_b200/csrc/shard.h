// Sharded batches: independent frames split over N GPUs (one process per GPU), finished frames
// gathered on rank 0 — the reference topology's last step is "frames reach the one display"
// (the reference's engine/NQ/fisheye.c:802-803 writes vid.buffer).  The gather of chunk k overlaps the
// warp of chunk k+1 (compute stream + communication stream per rank).
//   NCCL        ncclSend/ncclRecv of finished chunks (the north-star's "NCCL only for the final gather")
//   PEER_COPY   copy engines push finished chunks into rank 0's buffer through CUDA-IPC peer memory (NVLink)
//   PEER_STORE  the warp kernels store straight into rank 0's buffer (fused warp + gather)
// NCCL is loaded at run time (libnccl.so.2): the library has no link-time dependency on it.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace blinky {

class WarpDevice;

// contiguous block of frames owned by `rank`; block sizes differ by at most one
void shard_range(int total_frames, int rank, int world, int *first, int *count);

class ShardGroup {
public:
    static bool unique_id(unsigned char id[128], std::string &err);

    ShardGroup(WarpDevice *dev, int device);
    ~ShardGroup();
    bool init(int rank, int world, const unsigned char id[128]);
    // collective: rank 0 allocates total_frames x frame_bytes and shares it; *root_buffer = the buffer on rank 0, nullptr elsewhere
    bool buffer(int total_frames, size_t frame_bytes, void **root_buffer);
    bool warp_gather(const void *d_faces, size_t face_stride, int total_frames, int mode, int chunk_frames, void *stream);
    bool sync();
    const std::string &last_error() const { return err_; }
    int rank() const { return rank_; }
    int world() const { return world_; }

private:
    bool fail(const char *what, int cuda_err);
    bool nccl_fail(const char *what, int r);
    void release_buffer();

    WarpDevice *dev_;
    int device_;
    int rank_ = -1, world_ = 0;
    void *comm_ = nullptr;           // ncclComm_t
    void *compute_ = nullptr, *copy_ = nullptr;  // cudaStream_t
    std::vector<void *> events_;     // cudaEvent_t pool
    void *root_buf_ = nullptr;       // rank 0: the gather buffer; others: the IPC mapping of it
    size_t frame_bytes_ = 0;
    int total_frames_ = 0;
    uint8_t *stage_ = nullptr;       // peers: finished frames before they travel (NCCL / PEER_COPY)
    size_t stage_bytes_ = 0;
    uint8_t *token_ = nullptr;       // small device scratch (handle broadcast, completion tokens)
    std::string err_;
};

}  // namespace blinky
