// Host plumbing shared by the C-ABI units: the entry-point guard, device selection, device buffers kept until
// destroy, the fp32 weight upload, the weight table, the staging block, the GEMM dispatch, the session table and the
// state every engine handle holds.
#pragma once

#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/wlk_b200.h"
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

    // n floats -> dst as fp32 (a copy) or as dst_type (a conversion).  DT_BF16X2 puts the hi plane at dst and the lo
    // plane `plane` elements behind it; DT_E4M3 quantizes rows of `plane` columns, their scales to `scale`.  Synchronous:
    // `host` may be reused on return.
    void put(const float* host, size_t n, void* dst, int dst_type, cudaStream_t st, size_t plane = 0, float* scale = nullptr) {
        if (n > cap) {
            if (buf) { CUDA_CHECK(cudaStreamSynchronize(st)); CUDA_CHECK(cudaFree(buf)); }
            CUDA_CHECK(cudaMalloc(&buf, n * 4));
            cap = n;
        }
        CUDA_CHECK(cudaMemcpyAsync(buf, host, n * 4, cudaMemcpyHostToDevice, st));
        if (dst_type == DT_F32) CUDA_CHECK(cudaMemcpyAsync(dst, buf, n * 4, cudaMemcpyDeviceToDevice, st));
        else if (dst_type == DT_BF16X2) split_f32_to_planes(buf, (bf16*)dst, (bf16*)dst + plane, (int64_t)n, st);
        else if (dst_type == DT_E4M3)
            quantize_rows(buf, DT_F32, (int64_t)plane, (int)(n / plane), (int)plane, (uint8_t*)dst, (int64_t)plane, scale, st);
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

// An engine's weights.  At create the engine declares every checkpoint tensor once -- its name, its canonical shape and
// where its elements go -- together with the unnamed buffers it derives itself, then allocate() places them all in one
// device blob.  load() checks a tensor against its declaration by the engine's shape rule and uploads it; require_all()
// names the declared tensors that were not loaded.
struct WeightTable {
    // element count only; element count and leading axis (Conv kernels may carry trailing singleton axes); exact shape
    enum Rule { NUMEL, LEADING, EXACT };
    using Perm = std::function<std::vector<float>(const float* host)>;   // host rearrangement before the upload
    struct Dst {
        void** base;
        size_t off = 0;                  // element offset from *base (into the hi plane in DT_BF16X2)
        int type = DT_F32;
        size_t plane = 0;                // DT_BF16X2: elements from the hi plane to the lo plane (the whole matrix);
                                         // DT_E4M3: columns of a row
        Perm perm = nullptr;
        float** scale = nullptr;         // DT_E4M3: the matrix's row scales (row off / plane)
        template <typename T>
        Dst(T*& b, size_t o = 0, int t = DT_F32, size_t p = 0, Perm f = nullptr)
            : base(reinterpret_cast<void**>(&b)), off(o), type(t), plane(p), perm(std::move(f)) {}
    };
    struct Entry {
        std::string name;
        std::vector<int64_t> shape;
        std::vector<Dst> dst;            // none: accepted and dropped
        bool optional = false;
    };

    WeightUpload& up;
    cudaStream_t& st;
    Rule rule = EXACT;
    int wt = DT_F32;                     // type of the weight matrices
    std::vector<Entry> entries;          // in declaration order, the order require_all() reports in
    std::map<std::string, size_t> index;
    std::vector<std::pair<void**, size_t>> slots;   // pointer to set, byte offset in the blob
    size_t used = 0;
    uint8_t* blob = nullptr;
    size_t bytes = 0;
    std::set<std::string> loaded;

    // `nbytes` of the blob at the next 256-byte boundary; *slot points there once allocate() ran, so a slot must not
    // move in between (resize per-layer vectors before declaring)
    template <typename T>
    void buf(T*& slot, size_t nbytes) {
        used = (used + 255) / 256 * 256;
        slots.push_back({reinterpret_cast<void**>(&slot), used});
        used += nbytes;
    }
    Entry& add(const std::string& name, std::vector<int64_t> shape, std::vector<Dst> dst) {
        index[name] = entries.size();
        entries.push_back({name, std::move(shape), std::move(dst)});
        return entries.back();
    }
    // a tensor in a buffer of its own: an fp32 vector, or a matrix in the weight type
    Entry& f32(const std::string& name, float*& slot, std::vector<int64_t> shape) {
        buf(slot, (size_t)numel(shape.data(), (int)shape.size()) * 4);
        return add(name, std::move(shape), {Dst(slot)});
    }
    Entry& mat(const std::string& name, void*& slot, std::vector<int64_t> shape, Perm perm = nullptr) {
        const size_t n = (size_t)numel(shape.data(), (int)shape.size());
        buf(slot, n * dtype_size(wt));
        return add(name, std::move(shape), {Dst(slot, 0, wt, n, std::move(perm))});
    }
    // Tensors one after another in one buffer of `type`: [sum of rows][cols], or a vector when cols is 0.  A part without a
    // name is left zero.  DT_E4M3 (a matrix) also places its fp32 row scales at `scale`.
    template <typename T>
    void fused(T*& slot, int type, const std::vector<std::pair<std::string, int64_t>>& parts, int64_t cols,
               float** scale = nullptr) {
        int64_t rows = 0;
        for (auto& p : parts) rows += p.second;
        const size_t n = (size_t)rows * (cols ? cols : 1);
        buf(slot, n * dtype_size(type));
        if (type == DT_E4M3) buf(*scale, (size_t)rows * 4);
        int64_t r = 0;
        for (auto& p : parts) {
            if (!p.first.empty()) {
                Dst d(slot, (size_t)r * (cols ? cols : 1), type, type == DT_E4M3 ? (size_t)cols : n);
                d.scale = scale;
                add(p.first, cols ? std::vector<int64_t>{p.second, cols} : std::vector<int64_t>{p.second}, {d});
            }
            r += p.second;
        }
    }

    // The blob (with 256 bytes of tail slack), zero-filled, and every declared pointer into it.
    void allocate(DeviceAllocs& allocs, size_t* acct) {
        bytes = used + 256;
        blob = reinterpret_cast<uint8_t*>(allocs.take(bytes, acct));
        for (auto& s : slots) *s.first = blob + s.second;
    }

    void check_shape(const Entry& e, const int64_t* shape, int ndim) const {
        const int64_t n = numel(shape, ndim), want = numel(e.shape.data(), (int)e.shape.size());
        if (rule == NUMEL) {
            WLK_CHECK(n == want, "tensor %s has %lld elements, expected %lld", e.name.c_str(), (long long)n, (long long)want);
            return;
        }
        const bool ok = rule == LEADING ? n == want && shape[0] == e.shape[0]
                                        : std::vector<int64_t>(shape, shape + ndim) == e.shape;
        WLK_CHECK(ok, "tensor %s has the wrong shape for this geometry", e.name.c_str());
    }

    void load(const std::string& name, const float* host, const int64_t* shape, int ndim) {
        auto it = index.find(name);
        WLK_CHECK(it != index.end(), "unknown tensor %s", name.c_str());
        const Entry& e = entries[it->second];
        const int64_t n = numel(shape, ndim);
        if (!e.dst.empty()) check_shape(e, shape, ndim);      // an entry without a destination takes any shape
        for (const Dst& d : e.dst) {
            std::vector<float> tmp;
            if (d.perm) tmp = d.perm(host);
            uint8_t* dst = reinterpret_cast<uint8_t*>(*d.base) + d.off * (d.type == DT_F32 ? 4 : d.type == DT_E4M3 ? 1 : 2);
            float* scale = d.type == DT_E4M3 ? *d.scale + d.off / d.plane : nullptr;
            up.put(d.perm ? tmp.data() : host, d.perm ? tmp.size() : (size_t)n, dst, d.type, st, d.plane, scale);
        }
        loaded.insert(name);
    }

    // Every declared tensor that is not optional was loaded; the error names the first few that were not.
    void require_all() const {
        std::string missing;
        int nmiss = 0;
        for (auto& e : entries)
            if (!e.optional && !loaded.count(e.name) && nmiss++ < 5) missing += e.name + " ";
        WLK_CHECK(nmiss == 0, "%d tensors missing, e.g. %s", nmiss, missing.c_str());
    }
};

// [a][b][c] -> [a][c][b].  A Conv weight [Co][Ci][K] becomes tap-major [Co][K][Ci] (a tap's input channels are
// contiguous, like the im2col rows); a projection over channel-major features [d][C][F] reads [F][C] activations.
inline WeightTable::Perm swap_inner_axes(int64_t a, int64_t b, int64_t c) {
    return [=](const float* s) {
        std::vector<float> t((size_t)(a * b * c));
        for (int64_t i = 0; i < a; ++i)
            for (int64_t j = 0; j < b; ++j)
                for (int64_t k = 0; k < c; ++k) t[(size_t)((i * c + k) * b + j)] = s[(i * b + j) * c + k];
        return t;
    };
}

// "mel_filters" [n_mels][n_freq] (a Slaney filterbank): transposed to [n_freq][n_mels] at `filtT`, and the non-zero
// span [lo, hi) of every (triangular) filter at `span`.  The engine reserves both buffers.
inline WeightTable::Entry& declare_mel_filters(WeightTable& T, float*& filtT, int2*& span, int n_mels, int n_freq) {
    auto spans = [=](const float* s) {
        std::vector<float> out(2 * (size_t)n_mels);     // int2 per filter, carried bit for bit by the fp32 copy
        for (int m = 0; m < n_mels; ++m) {
            int lo = n_freq, hi = 0;
            for (int k = 0; k < n_freq; ++k)
                if (s[(size_t)m * n_freq + k] != 0.f) { if (k < lo) lo = k; hi = k + 1; }
            if (lo >= hi) { lo = 0; hi = 0; }
            const int2 v = make_int2(lo, hi);
            memcpy(&out[2 * (size_t)m], &v, sizeof(v));
        }
        return out;
    };
    return T.add("mel_filters", {n_mels, n_freq},
                 {WeightTable::Dst(filtT, 0, DT_F32, 0, swap_inner_axes(1, n_mels, n_freq)),
                  WeightTable::Dst(span, 0, DT_F32, 0, spans)});
}

// A pinned host block mirrored on the device: a call lays out its small per-call arrays (jobs, row maps, pointer
// tables) in it with a Stager and sends them in one H2D copy.  The event recorded after that copy guards the host
// block: the next layout waits on it before it writes.
struct Staging {
    uint8_t *host = nullptr, *dev = nullptr;
    size_t bytes = 0;
    cudaEvent_t done = nullptr;

    void alloc(size_t n, DeviceAllocs& allocs, size_t* acct) {
        bytes = n;
        CUDA_CHECK(cudaMallocHost(&host, n));
        dev = reinterpret_cast<uint8_t*>(allocs.take(n, acct));
        CUDA_CHECK(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
    }
    void release() {                                     // `dev` belongs to the DeviceAllocs
        if (host) cudaFreeHost(host);
        if (done) cudaEventDestroy(done);
        host = nullptr;
        done = nullptr;
    }
};

// One layout of the staging block.  Arrays go in call order, each at a 256-byte-aligned offset, so the same sequence of
// sizes always gives the same device pointers (captured CUDA graphs replay them).
struct Stager {
    Staging& stg;
    size_t used = 0;
    explicit Stager(Staging& s) : stg(s) { CUDA_CHECK(cudaEventSynchronize(stg.done)); }
    template <typename T>
    T* host(size_t count, T** dev) {
        size_t off = (used + 255) / 256 * 256;
        size_t bytes = count * sizeof(T);
        WLK_CHECK(off + bytes <= stg.bytes, "staging buffer overflow (%zu + %zu > %zu)", off, bytes, stg.bytes);
        used = off + bytes;
        *dev = reinterpret_cast<T*>(stg.dev + off);
        return reinterpret_cast<T*>(stg.host + off);
    }
    void upload(cudaStream_t st) {
        if (used) CUDA_CHECK(cudaMemcpyAsync(stg.dev, stg.host, used, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaEventRecord(stg.done, st));
    }
};

// An engine's GEMM launch: the split-K scratch of the wgmma kernels and the choice between them and the SIMT kernel.
// Each engine decides by its own rule whether a GEMM should run on the tensor cores and passes the result as `tc`.
struct GemmDispatch {
    float* sk_scratch = nullptr;
    int* sk_counters = nullptr;

    // Taken only by an engine that runs wgmma GEMMs.
    void alloc(DeviceAllocs& allocs, size_t* acct) {
        sk_scratch = (float*)allocs.take(SK_SCRATCH_FLOATS * sizeof(float), acct);
        sk_counters = (int*)allocs.take(SK_MAX_TILES * sizeof(int), acct);
    }
    void wire(GemmArgs& g) const {
        g.sk_scratch = sk_scratch; g.sk_scratch_floats = SK_SCRATCH_FLOATS;
        g.sk_counters = sk_counters; g.sk_max_tiles = SK_MAX_TILES;
    }
    // A shape the wgmma kernels do not take runs on the SIMT kernel, unless `strict` names the caller: then it raises.
    void run(GemmArgs& g, bool tc, cudaStream_t st, int num_sms, const char* strict = nullptr) const {
        if (g.M <= 0) return;
        wire(g);
        if (tc) {
            std::string why;
            if (gemm_tcgen05_supported(g, strict ? &why : nullptr)) { gemm_tcgen05(g, st, num_sms); return; }
            WLK_CHECK(!strict, "%s GEMM %dx%dx%d has no wgmma kernel: %s", strict, g.M, g.N, g.K, why.c_str());
        }
        gemm_simt(g, st);
    }
};

// An engine's session slots.  S has a `bool open`; a closed slot is free.
template <typename S>
struct SessionTable {
    std::vector<S> slots;

    int size() const { return (int)slots.size(); }
    S& operator[](int32_t sid) { return slots[sid]; }    // a sid that at() or check_batch() accepted
    typename std::vector<S>::iterator begin() { return slots.begin(); }
    typename std::vector<S>::iterator end() { return slots.end(); }

    int free_slot() const {
        for (int i = 0; i < size(); ++i)
            if (!slots[i].open) return i;
        WLK_CHECK(false, "all %d sessions in use", size());
        return -1;
    }
    S& at(int32_t sid) {
        WLK_CHECK(sid >= 0 && sid < size() && slots[sid].open, "invalid session id %d", sid);
        return slots[sid];
    }
    // Every sid of a batch names an open session, and none appears twice.
    void check_batch(const int32_t* sids, int n) {
        for (int i = 0; i < n; ++i) {
            at(sids[i]);
            for (int j = 0; j < i; ++j) WLK_CHECK(sids[j] != sids[i], "session %d appears twice in the batch", sids[i]);
        }
    }
};

// What every engine handle holds.  Calls on a handle take `mu` and make cfg.device current (WLK_ENTER).
struct EngineBase {
    wlk_config cfg{};
    int act = DT_F32;                    // activation type
    int num_sms = 132;
    cudaStream_t st = nullptr;
    std::mutex mu;
    DeviceAllocs allocs;                 // buffers kept from create (or first use) until destroy
    WeightUpload upload;
    WeightTable weights{upload, st};
    size_t bytes_weights = 0, bytes_sessions = 0, bytes_workspace = 0;
    bool finalized = false;
    Staging stg;
    GemmDispatch gemm;

    size_t es() const { return dtype_size(act); }

    // The device (sm_90a only), then the engine's non-blocking stream.
    void open(const wlk_config& c) {
        cfg = c;
        num_sms = open_sm90_device(c.device);
        CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    }
    // Waits for the stream, lets the engine free its sessions and its own buffers, then frees what every engine holds.
    template <typename F>
    void close(F&& free_own) {
        cudaStreamSynchronize(st);
        free_own();
        allocs.free_all();
        upload.release();
        stg.release();
        cudaStreamDestroy(st);
    }
    void memory(size_t* weights, size_t* sessions, size_t* workspace) const {
        if (weights) *weights = bytes_weights;
        if (sessions) *sessions = bytes_sessions;
        if (workspace) *workspace = bytes_workspace;
    }
};

}  // namespace wlk
