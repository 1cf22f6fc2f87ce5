// One owned cudaMalloc allocation, freed with cudaFree when its owner goes.  CUDA types are kept out of this header
// (plain C++ translation units include it through warp_device.h); the out-of-line parts are in warp_device.cu.
#pragma once

#include <cstddef>
#include <utility>

namespace blinky {

class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(DeviceBuffer &&o) noexcept : p_(o.p_) { o.p_ = nullptr; }
    DeviceBuffer &operator=(DeviceBuffer &&o) noexcept {
        std::swap(p_, o.p_);  // (o frees what this buffer held)
        return *this;
    }
    DeviceBuffer(const DeviceBuffer &) = delete;
    DeviceBuffer &operator=(const DeviceBuffer &) = delete;
    ~DeviceBuffer() { reset(); }

    // frees what the buffer held and allocates `bytes` on the current device; the cudaError_t (0: success)
    int alloc(size_t bytes);
    void reset();
    void *get() const { return p_; }
    template <typename T>
    T *as() const { return static_cast<T *>(p_); }

private:
    void *p_ = nullptr;
};

}  // namespace blinky
