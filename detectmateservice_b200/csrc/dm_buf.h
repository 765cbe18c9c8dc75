// dm_buf.h -- owners of the CUDA runtime objects libdmdetect creates (host only; not part of the CPU emulator).
//
// Each owner frees its object exactly once: when it is destroyed, grown, reset or moved onto.  An empty owner frees
// nothing.  This is the only file of csrc/ that allocates or destroys runtime objects.
#pragma once
#include <cstring>
#include <memory>
#include <utility>
#include <cuda_runtime.h>

struct DmDeviceMem {
    void operator()(void* p) const { cudaFree(p); }
    static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
    static cudaError_t zero(void* p, size_t bytes) { return cudaMemset(p, 0, bytes); }
};

template <unsigned Flags>
struct DmPinnedMem {
    void operator()(void* p) const { cudaFreeHost(p); }
    static cudaError_t alloc(void** p, size_t bytes) { return cudaHostAlloc(p, bytes, Flags); }
    static cudaError_t zero(void* p, size_t bytes) { memset(p, 0, bytes); return cudaSuccess; }
};

// A buffer of cap() elements of T.
template <typename T, typename Mem>
class DmBuf {
  public:
    DmBuf() = default;
    DmBuf(DmBuf&& o) noexcept : p_(std::move(o.p_)), cap_(std::exchange(o.cap_, 0)) {}
    DmBuf& operator=(DmBuf&& o) noexcept {
        p_ = std::move(o.p_);
        cap_ = std::exchange(o.cap_, 0);
        return *this;
    }

    // Holds at least need elements afterwards: does nothing when it already does, else frees the old allocation (its
    // contents are not kept) and allocates grow_to elements, zeroed if asked.  A failed allocation leaves the owner
    // empty, with capacity 0, and is returned.
    cudaError_t grow(size_t need, size_t grow_to, bool zero = false) {
        if (need <= cap_) return cudaSuccess;
        reset();
        void* p = nullptr;
        cudaError_t e = Mem::alloc(&p, grow_to * sizeof(T));
        if (e == cudaSuccess) p_.reset(static_cast<T*>(p));
        if (e == cudaSuccess && zero) e = Mem::zero(p, grow_to * sizeof(T));
        if (e == cudaSuccess) cap_ = grow_to;
        else p_.reset();
        return e;
    }
    cudaError_t alloc(size_t n, bool zero = false) { return grow(n, n, zero); }   // n elements, allocated once
    void reset() { p_.reset(); cap_ = 0; }

    T* get() const { return p_.get(); }
    size_t cap() const { return cap_; }

  private:
    std::unique_ptr<T, Mem> p_;
    size_t cap_ = 0;
};

template <typename T>
using DmDev = DmBuf<T, DmDeviceMem>;
template <typename T, unsigned Flags = cudaHostAllocDefault>
using DmPinned = DmBuf<T, DmPinnedMem<Flags>>;

struct DmDestroy {
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};

// An event or a stream.  create() replaces what the owner held; on failure it is left empty.
template <typename S, cudaError_t (*Create)(S**, unsigned), unsigned Flags>
struct DmObj : std::unique_ptr<S, DmDestroy> {
    cudaError_t create(unsigned flags = Flags) {
        S* v = nullptr;
        const cudaError_t e = Create(&v, flags);
        this->reset(e == cudaSuccess ? v : nullptr);
        return e;
    }
};
using DmEvent = DmObj<CUevent_st, cudaEventCreateWithFlags, cudaEventDisableTiming>;
using DmStream = DmObj<CUstream_st, cudaStreamCreateWithFlags, cudaStreamNonBlocking>;   // not ordered behind the legacy stream

// Puts a configuration struct on the device: d's one T is allocated once, and the blocking copy waits for `after`
// first.  Pass the handle's last stream: a copy on the legacy stream does not order against the handle's non-blocking
// streams, so a kernel still in flight there could read the struct while it is overwritten.
template <typename T>
static inline cudaError_t dm_upload(DmDev<T>& d, const T& v, cudaStream_t after) {
    cudaError_t e = d.alloc(1);
    if (e == cudaSuccess) e = cudaStreamSynchronize(after);
    if (e == cudaSuccess) e = cudaMemcpy(d.get(), &v, sizeof(T), cudaMemcpyHostToDevice);
    return e;
}
