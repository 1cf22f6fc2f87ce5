#include "shard.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types only: every entry point is looked up with dlsym

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "../../include/blinky_b200.h"
#include "warp_device.h"

namespace blinky {

void shard_range(int total_frames, int rank, int world, int *first, int *count) {
    if (world < 1) world = 1;
    if (total_frames < 0) total_frames = 0;
    const int base = total_frames / world, extra = total_frames % world;
    if (first) *first = rank * base + std::min(rank, extra);
    if (count) *count = base + (rank < extra ? 1 : 0);
}

namespace {

struct Nccl {
    void *lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    std::string why;
};

Nccl &nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *names[] = {getenv("BLINKY_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char *nm : names) {
            if (!nm || !*nm) continue;
            n.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (n.lib) break;
        }
        if (!n.lib) {
            n.why = std::string("cannot load NCCL (libnccl.so.2; set BLINKY_NCCL_LIB): ") + (dlerror() ? dlerror() : "");
            return;
        }
#define SYM(field, name)                                                        \
    n.field = reinterpret_cast<decltype(n.field)>(dlsym(n.lib, name));          \
    if (!n.field && n.why.empty()) n.why = std::string("NCCL symbol missing: ") + name;
        SYM(GetUniqueId, "ncclGetUniqueId")
        SYM(CommInitRank, "ncclCommInitRank")
        SYM(CommDestroy, "ncclCommDestroy")
        SYM(Send, "ncclSend")
        SYM(Recv, "ncclRecv")
        SYM(Broadcast, "ncclBroadcast")
        SYM(GroupStart, "ncclGroupStart")
        SYM(GroupEnd, "ncclGroupEnd")
        SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
    });
    return n;
}

}  // namespace

#define CK(call)                                       \
    do {                                               \
        cudaError_t e_ = (call);                       \
        if (e_ != cudaSuccess) return fail(#call, e_); \
    } while (0)
#define NK(call)                                          \
    do {                                                  \
        ncclResult_t r_ = (call);                         \
        if (r_ != ncclSuccess) return nccl_fail(#call, r_); \
    } while (0)

bool ShardGroup::fail(const char *what, int cuda_err) {
    err_ = std::string(what) + ": " + cudaGetErrorString(static_cast<cudaError_t>(cuda_err));
    return false;
}

bool ShardGroup::nccl_fail(const char *what, int r) {
    Nccl &n = nccl();
    err_ = std::string(what) + ": " + (n.GetErrorString ? n.GetErrorString(static_cast<ncclResult_t>(r)) : "NCCL error");
    return false;
}

bool ShardGroup::unique_id(unsigned char id[128], std::string &err) {
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    Nccl &n = nccl();
    if (!n.why.empty()) {
        err = n.why;
        return false;
    }
    ncclUniqueId u;
    ncclResult_t r = n.GetUniqueId(&u);
    if (r != ncclSuccess) {
        err = std::string("ncclGetUniqueId: ") + n.GetErrorString(r);
        return false;
    }
    memcpy(id, &u, 128);
    return true;
}

ShardGroup::ShardGroup(WarpDevice *dev, int device) : dev_(dev), device_(device) {}

ShardGroup::~ShardGroup() {
    cudaSetDevice(device_);
    cudaDeviceSynchronize();
    release_buffer();
    cudaFree(stage_);
    cudaFree(token_);
    for (void *e : events_) cudaEventDestroy(static_cast<cudaEvent_t>(e));
    if (compute_) cudaStreamDestroy(static_cast<cudaStream_t>(compute_));
    if (copy_) cudaStreamDestroy(static_cast<cudaStream_t>(copy_));
    if (comm_) nccl().CommDestroy(static_cast<ncclComm_t>(comm_));
}

void ShardGroup::release_buffer() {
    if (!root_buf_) return;
    if (rank_ == 0) cudaFree(root_buf_);
    else cudaIpcCloseMemHandle(root_buf_);
    root_buf_ = nullptr;
}

bool ShardGroup::init(int rank, int world, const unsigned char id[128]) {
    if (comm_) {
        err_ = "shard group already initialised";
        return false;
    }
    if (world < 1 || rank < 0 || rank >= world) {
        err_ = "shard init: bad rank/world";
        return false;
    }
    Nccl &n = nccl();
    if (!n.why.empty()) {
        err_ = n.why;
        return false;
    }
    CK(cudaSetDevice(device_));
    ncclUniqueId u;
    memcpy(&u, id, 128);
    ncclComm_t c;
    NK(n.CommInitRank(&c, world, u, rank));
    comm_ = c;
    rank_ = rank;
    world_ = world;
    cudaStream_t s;
    CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    compute_ = s;
    CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    copy_ = s;
    CK(cudaMalloc(&token_, 256));
    CK(cudaMemset(token_, 0, 256));
    return true;
}

bool ShardGroup::buffer(int total_frames, size_t frame_bytes, void **root_buffer) {
    if (!comm_) {
        err_ = "shard buffer: call blinky_shard_init first";
        return false;
    }
    Nccl &n = nccl();
    CK(cudaSetDevice(device_));
    CK(cudaDeviceSynchronize());
    release_buffer();
    const size_t bytes = static_cast<size_t>(total_frames) * frame_bytes;
    cudaStream_t cs = static_cast<cudaStream_t>(copy_);
    cudaIpcMemHandle_t h;
    memset(&h, 0, sizeof h);
    if (rank_ == 0) {
        CK(cudaMalloc(&root_buf_, bytes ? bytes : 1));
        CK(cudaIpcGetMemHandle(&h, root_buf_));
        CK(cudaMemcpyAsync(token_, &h, sizeof h, cudaMemcpyHostToDevice, cs));
    }
    if (world_ > 1) NK(n.Broadcast(token_, token_, sizeof h, ncclUint8, 0, static_cast<ncclComm_t>(comm_), cs));
    CK(cudaStreamSynchronize(cs));
    if (rank_ != 0) {
        CK(cudaMemcpy(&h, token_, sizeof h, cudaMemcpyDeviceToHost));
        // maps rank 0's buffer into this process: stores and copies to it travel over NVLink
        CK(cudaIpcOpenMemHandle(&root_buf_, h, cudaIpcMemLazyEnablePeerAccess));
    }
    frame_bytes_ = frame_bytes;
    total_frames_ = total_frames;
    if (root_buffer) *root_buffer = rank_ == 0 ? root_buf_ : nullptr;
    return true;
}

bool ShardGroup::warp_gather(const void *d_faces, size_t face_stride, int total_frames, int mode, int chunk_frames, void *stream) {
    if (!comm_ || !root_buf_) {
        err_ = "shard warp_gather: call blinky_shard_init and blinky_shard_buffer first";
        return false;
    }
    if (total_frames != total_frames_) {
        err_ = "shard warp_gather: total_frames differs from the shared buffer's";
        return false;
    }
    if (mode != BLINKY_GATHER_NCCL && mode != BLINKY_GATHER_PEER_COPY && mode != BLINKY_GATHER_PEER_STORE) {
        err_ = "shard warp_gather: unknown mode";
        return false;
    }
    Nccl &n = nccl();
    CK(cudaSetDevice(device_));
    ncclComm_t comm = static_cast<ncclComm_t>(comm_);
    cudaStream_t user = static_cast<cudaStream_t>(stream), comp = static_cast<cudaStream_t>(compute_), cpy = static_cast<cudaStream_t>(copy_);
    int first = 0, count = 0;
    shard_range(total_frames, rank_, world_, &first, &count);
    if (chunk_frames < 1) chunk_frames = 1;
    const int nch = (count + chunk_frames - 1) / chunk_frames;
    int max_nch = 0;
    for (int r = 0; r < world_; ++r) {
        int f, c;
        shard_range(total_frames, r, world_, &f, &c);
        max_nch = std::max(max_nch, (c + chunk_frames - 1) / chunk_frames);
    }
    // events: [0] inputs ready, [1..nch] chunk warped, [nch+1] compute done, [nch+2] copy done
    const size_t need = static_cast<size_t>(nch) + 3;
    while (events_.size() < need) {
        cudaEvent_t e;
        CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        events_.push_back(e);
    }
    auto ev = [&](size_t i) { return static_cast<cudaEvent_t>(events_[i]); };
    CK(cudaEventRecord(ev(0), user));
    CK(cudaStreamWaitEvent(comp, ev(0), 0));
    CK(cudaStreamWaitEvent(cpy, ev(0), 0));
    const uint8_t *faces = static_cast<const uint8_t *>(d_faces);
    uint8_t *root = static_cast<uint8_t *>(root_buf_);
    const size_t fb = frame_bytes_;

    if (rank_ != 0 && mode != BLINKY_GATHER_PEER_STORE) {
        const size_t want = static_cast<size_t>(count) * fb;
        if (want > stage_bytes_) {
            CK(cudaDeviceSynchronize());
            cudaFree(stage_);
            stage_ = nullptr;
            CK(cudaMalloc(&stage_, want));
            stage_bytes_ = want;
        }
    }
    for (int c = 0; c < max_nch; ++c) {
        if (c < nch) {
            const int f0 = c * chunk_frames, nf = std::min(chunk_frames, count - f0);
            // rank 0 and PEER_STORE: the kernel writes the frames where they belong in rank 0's buffer
            uint8_t *out = (rank_ == 0 || mode == BLINKY_GATHER_PEER_STORE) ? root + static_cast<size_t>(first + f0) * fb : stage_ + static_cast<size_t>(f0) * fb;
            if (!dev_->warp(WarpRequest(faces + static_cast<size_t>(f0) * face_stride, face_stride, out, fb, nf, comp))) {
                err_ = dev_->last_error();
                return false;
            }
            CK(cudaEventRecord(ev(1 + static_cast<size_t>(c)), comp));
            if (rank_ != 0 && mode != BLINKY_GATHER_PEER_STORE) {
                CK(cudaStreamWaitEvent(cpy, ev(1 + static_cast<size_t>(c)), 0));
                if (mode == BLINKY_GATHER_NCCL) {
                    NK(n.Send(out, static_cast<size_t>(nf) * fb, ncclUint8, 0, comm, cpy));
                } else {
                    CK(cudaMemcpyAsync(root + static_cast<size_t>(first + f0) * fb, out, static_cast<size_t>(nf) * fb, cudaMemcpyDeviceToDevice, cpy));
                }
            }
        }
        if (rank_ == 0 && mode == BLINKY_GATHER_NCCL && world_ > 1) {
            NK(n.GroupStart());
            for (int r = 1; r < world_; ++r) {
                int rf, rc;
                shard_range(total_frames, r, world_, &rf, &rc);
                const int f0 = c * chunk_frames, nf = std::min(chunk_frames, rc - f0);
                if (nf > 0) NK(n.Recv(root + static_cast<size_t>(rf + f0) * fb, static_cast<size_t>(nf) * fb, ncclUint8, r, comm, cpy));
            }
            NK(n.GroupEnd());
        }
    }
    // peer modes: one byte per peer tells rank 0 that the peer's writes have landed
    if (mode != BLINKY_GATHER_NCCL && world_ > 1) {
        if (rank_ == 0) {
            NK(n.GroupStart());
            for (int r = 1; r < world_; ++r) NK(n.Recv(token_ + 64 + r, 1, ncclUint8, r, comm, cpy));
            NK(n.GroupEnd());
        } else {
            if (nch > 0) CK(cudaStreamWaitEvent(cpy, ev(static_cast<size_t>(nch)), 0));
            NK(n.Send(token_ + 64, 1, ncclUint8, 0, comm, cpy));
        }
    }
    CK(cudaEventRecord(ev(static_cast<size_t>(nch) + 1), comp));
    CK(cudaEventRecord(ev(static_cast<size_t>(nch) + 2), cpy));
    CK(cudaStreamWaitEvent(user, ev(static_cast<size_t>(nch) + 1), 0));
    CK(cudaStreamWaitEvent(user, ev(static_cast<size_t>(nch) + 2), 0));
    return true;
}

bool ShardGroup::sync() {
    CK(cudaSetDevice(device_));
    CK(cudaStreamSynchronize(static_cast<cudaStream_t>(compute_)));
    CK(cudaStreamSynchronize(static_cast<cudaStream_t>(copy_)));
    return true;
}

}  // namespace blinky
