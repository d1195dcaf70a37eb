// Host plumbing shared by the C-ABI units: the entry-point guard, device selection, device buffers kept until
// destroy, the fp32 weight upload and the checks on loaded tensors.
#pragma once

#include <initializer_list>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "kernels.cuh"

// The body of every extern "C" entry point runs between these.  No exception crosses the C ABI: the message goes to
// wlk_last_error() and the return code says what was thrown (0 nothing, 1 wlk::Error, 2 std::exception, 3 other).
#define WLK_API_BEGIN try {
#define WLK_API_END                                                  \
    return 0;                                                        \
    } catch (const wlk::Error& err) {                                \
        wlk::set_last_error(err.msg);                                \
        return 1;                                                    \
    } catch (const std::exception& ex) {                             \
        wlk::set_last_error(std::string("exception: ") + ex.what()); \
        return 2;                                                    \
    } catch (...) {                                                  \
        wlk::set_last_error("unknown exception");                    \
        return 3;                                                    \
    }

// Entry of a call on an engine handle: reject a null handle, hold the engine's mutex for the rest of the call and make
// its device current.
#define WLK_ENTER(h, device)                                  \
    WLK_CHECK((h) != nullptr, "null engine");                 \
    std::lock_guard<std::mutex> _lk((h)->mu);                 \
    CUDA_CHECK(cudaSetDevice(device))

namespace wlk {

inline void use_device(int device) {
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    WLK_CHECK(ce == cudaSuccess && ndev > 0, "no CUDA device available (%s): the library has no CPU fallback",
              cudaGetErrorString(ce));
    WLK_CHECK(device >= 0 && device < ndev, "device %d out of range (%d devices)", device, ndev);
    CUDA_CHECK(cudaSetDevice(device));
}

// use_device() for an engine: the library holds sm_90a code only.  Returns the device's SM count.
inline int open_sm90_device(int device) {
    use_device(device);
    cudaDeviceProp prop;
    CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    WLK_CHECK(prop.major == 9 && prop.minor == 0, "this library contains sm_90a code only; device %d is sm_%d%d", device,
              prop.major, prop.minor);
    return prop.multiProcessorCount;
}

// Device buffers an engine keeps until it is destroyed.
struct DeviceAllocs {
    std::vector<void*> ptrs;

    // At least 16 bytes, zero-filled.  The fill is complete when take() returns, so the buffer may be written from any
    // stream (the engines' streams do not synchronize with the default stream the fill runs on).  The size is added to
    // *acct when acct is given.
    void* take(size_t bytes, size_t* acct) {
        if (bytes < 16) bytes = 16;
        void* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, bytes));
        ptrs.push_back(p);
        CUDA_CHECK(cudaMemset(p, 0, bytes));
        CUDA_CHECK(cudaStreamSynchronize(0));
        if (acct) *acct += bytes;
        return p;
    }
    void free_all() {
        for (void* p : ptrs) cudaFree(p);
        ptrs.clear();
    }
};

// Upload of host fp32 tensors through a device staging buffer that only grows until release().
struct WeightUpload {
    float* buf = nullptr;
    size_t cap = 0;

    // n floats -> dst as fp32 (a copy) or as dst_type (a conversion).  Synchronous: `host` may be reused on return.
    void put(const float* host, size_t n, void* dst, int dst_type, cudaStream_t st) {
        if (n > cap) {
            if (buf) { CUDA_CHECK(cudaStreamSynchronize(st)); CUDA_CHECK(cudaFree(buf)); }
            CUDA_CHECK(cudaMalloc(&buf, n * 4));
            cap = n;
        }
        CUDA_CHECK(cudaMemcpyAsync(buf, host, n * 4, cudaMemcpyHostToDevice, st));
        if (dst_type == DT_F32) CUDA_CHECK(cudaMemcpyAsync(dst, buf, n * 4, cudaMemcpyDeviceToDevice, st));
        else convert_f32_to(buf, dst, dst_type, (int64_t)n, st);
        CUDA_CHECK(cudaStreamSynchronize(st));
    }
    void release() {
        if (buf) cudaFree(buf);
        buf = nullptr;
        cap = 0;
    }
};

// Device copies of an op-level call's host index arrays, freed once the op's work on the stream is done.
struct OpUpload {
    cudaStream_t st;
    std::vector<void*> bufs;
    template <typename X>
    const X* put(const X* host, size_t n) {
        void* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, (n > 1 ? n : 1) * sizeof(X)));
        bufs.push_back(p);
        CUDA_CHECK(cudaMemcpyAsync(p, host, n * sizeof(X), cudaMemcpyHostToDevice, st));
        return (const X*)p;
    }
    ~OpUpload() {
        cudaStreamSynchronize(st);
        for (void* p : bufs) cudaFree(p);
    }
};

inline int64_t numel(const int64_t* shape, int ndim) {
    int64_t n = 1;
    for (int i = 0; i < ndim; ++i) n *= shape[i];
    return n;
}

// The tensor's shape must be exactly `want`.
inline void expect_shape(const char* name, const int64_t* shape, int ndim, std::initializer_list<int64_t> want) {
    bool ok = (int)want.size() == ndim;
    int i = 0;
    for (int64_t w : want) { if (ok && shape[i] != w) ok = false; ++i; }
    WLK_CHECK(ok, "tensor %s has the wrong shape for this geometry", name);
}

// Every name in `required` must have been loaded; the error names the first few that were not.
inline void require_loaded(const std::set<std::string>& loaded, const std::vector<std::string>& required) {
    std::string missing;
    int nmiss = 0;
    for (auto& r : required)
        if (!loaded.count(r) && nmiss++ < 5) missing += r + " ";
    WLK_CHECK(nmiss == 0, "%d tensors missing, e.g. %s", nmiss, missing.c_str());
}

}  // namespace wlk
