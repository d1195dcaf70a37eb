// Shared declarations for the streaming-Whisper engine (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>

namespace wlk {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------
// errors: every C-ABI entry catches and stores a thread-local message
// ---------------------------------------------------------------------------------
void set_last_error(const std::string& msg);

struct Error {
    std::string msg;
};

#define WLK_CHECK(cond, ...)                                                                   \
    do {                                                                                       \
        if (!(cond)) {                                                                         \
            char _b[512];                                                                      \
            snprintf(_b, sizeof(_b), __VA_ARGS__);                                             \
            throw ::wlk::Error{std::string(_b) + " [" #cond " @ " __FILE__ ":" +               \
                               std::to_string(__LINE__) + "]"};                                \
        }                                                                                      \
    } while (0)

#define CUDA_CHECK(expr)                                                                       \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess)                                                                 \
            throw ::wlk::Error{std::string("CUDA error: ") + cudaGetErrorString(_e) +          \
                               " in " #expr " @ " __FILE__ ":" + std::to_string(__LINE__)};    \
    } while (0)

// ---------------------------------------------------------------------------------
// Programmatic dependent launch for the decoder's chains of short kernels: the next kernel's CTAs become
// resident (and run their prologue -- barrier init, weight-panel TMA) while the previous
// kernel drains.  Contract: a kernel launched through launch_pdl() executes ptx::griddep_wait() before it
// touches anything an earlier kernel produced (or still reads), so completion stays transitive along the
// chain; WLK_PDL=0 turns the attribute off (plain stream order).
// ---------------------------------------------------------------------------------
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// True the first time it is called for the current device with this flag array: kernel attributes (dynamic shared
// memory limits) and scratch allocations are per device, and several engines -- one per GPU -- may live in a process.
inline bool first_on_device(bool (&seen)[64]) {
    static std::mutex mu;                       // engines on different threads may race to the first launch
    int d = 0;
    cudaGetDevice(&d);
    d &= 63;
    std::lock_guard<std::mutex> lk(mu);
    if (seen[d]) return false;
    seen[d] = true;
    return true;
}
inline int current_device() { int d = 0; cudaGetDevice(&d); return d & 63; }

// DT_BF16X2: weights of the WLK_PREC_BF16X3 mode -- two bf16 planes (hi, then lo right behind it), 4 bytes per element
enum DType { DT_F32 = 0, DT_BF16 = 1, DT_BF16X2 = 2 };
inline size_t dtype_size(int t) { return t == DT_BF16 ? 2 : 4; }

// ---------------------------------------------------------------------------------
// GEMM epilogue description shared by the SIMT and the tensor-core GEMM kernels.
//   v = acc + bias[n];  v = act(v) (gelu: 1 erf-GELU, 2 ReLU, 3 SiLU);  if n < scale_cols: v *= col_scale;
//   if residual: v += residual[m, n];   then stored according to `mode`.
// ---------------------------------------------------------------------------------
enum EpiMode {
    EPI_PLAIN = 0,       // C[m * ldc + n]
    EPI_XKV = 1,         // cross-K/V head-major scatter: see engine.cu (cross_kv layout)
    EPI_SELF_QKV = 2,    // decoder self-attn: q -> plain buffer, k/v -> self-KV cache via row map
    EPI_ROWPTR = 3,      // C row pointers per batch: row m -> batch_ptrs[m / rows_per_batch] + (m % rpb) * ldc
};

struct Epilogue {
    const float* bias = nullptr;     // [N] fp32 or null
    int gelu = 0;                    // activation: 0 none, 1 erf-GELU, 2 ReLU, 3 SiLU (x * sigmoid x)
    float col_scale = 1.f;
    int scale_cols = 0;              // columns [0, scale_cols) are multiplied by col_scale ...
    int scale_period = 0;            // ... taken modulo scale_period when it is non-zero
    const float* residual = nullptr; // fp32 [M, ldr] (may alias C when c_type == fp32)
    int64_t ldr = 0;
    void* C = nullptr;
    int c_type = DT_F32;
    int64_t ldc = 0;
    int mode = EPI_PLAIN;
    // scatter parameters
    void* const* batch_ptrs = nullptr;   // EPI_XKV / EPI_ROWPTR / EPI_SELF_QKV: per-slot base pointers
    int rows_per_batch = 1;              // EPI_XKV / EPI_ROWPTR
    int rows_valid = 1 << 30;            // EPI_ROWPTR: rows with (m % rows_per_batch) >= rows_valid are dropped;
                                         //             the residual is indexed by the in-batch row
    int n_head = 0, d_model = 0;         // head-major scatters
    int kv_len = 0;                      // rows per (layer,kv,head) plane: 1500 (cross) / n_text_ctx (self)
    int layer = 0;                       // EPI_SELF_QKV
    const int32_t* row_slot = nullptr;   // EPI_SELF_QKV (and EPI_XKV when set): row -> index into batch_ptrs
    const int32_t* row_pos = nullptr;    // EPI_SELF_QKV (and EPI_XKV when set): row -> row of the K/V plane
};

struct GemmArgs {
    const void* A = nullptr; int a_type = DT_F32; int64_t lda = 0;   // [M, K] row-major (K contiguous)
    const void* W = nullptr; int w_type = DT_F32; int64_t ldw = 0;   // [N, K] row-major (K contiguous)
    const void* W_lo = nullptr;          // DT_BF16X2: the lo plane (W is the hi plane)
    void* a_split = nullptr;             // DT_BF16X2: scratch for the (hi, lo) planes of the fp32 A operand,
    size_t a_split_elems = 0;            //            a_split_elems bf16 per plane
    int M = 0, N = 0, K = 0;
    Epilogue epi;
    // split-K workspace of the CALLING engine (its stream orders the launches that share it): fp32 partial tiles and
    // one arrival counter per output tile, zero between launches.  Null: the GEMM runs unsplit.
    float* sk_scratch = nullptr; size_t sk_scratch_floats = 0;
    int* sk_counters = nullptr; int sk_max_tiles = 0;
};
constexpr size_t SK_SCRATCH_FLOATS = (size_t)8 << 20;     // 32 MB per engine
constexpr int SK_MAX_TILES = 4096;

void gemm_simt(const GemmArgs& g, cudaStream_t st);
void gemm_tcgen05(const GemmArgs& g, cudaStream_t st, int num_sms, int variant = 0);   // 0 auto, 1 64-wide tiles, 2 128-wide tiles
bool gemm_tcgen05_supported(const GemmArgs& g, std::string* why);

// ---------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ float gelu_erf(float x) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f32<bf16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Apply the arithmetic part of the epilogue to one accumulator element.
__device__ __forceinline__ float epi_math(const Epilogue& e, float v, int m, int n) {
    if (e.bias) v += __ldg(e.bias + n);
    if (e.gelu == 1) v = gelu_erf(v);
    else if (e.gelu == 2) v = fmaxf(v, 0.f);
    else if (e.gelu == 3) v = v / (1.0f + expf(-v));
    if ((e.scale_period ? (n % e.scale_period) : n) < e.scale_cols) v *= e.col_scale;
    if (e.residual) {
        int rr = (e.mode == EPI_ROWPTR) ? (m % e.rows_per_batch) : m;
        v += e.residual[(int64_t)rr * e.ldr + n];
    }
    return v;
}

// Destination address (in elements of the output type) for element (m, n); nullptr-safe
// callers must have checked m < M, n < N.  Returns the base pointer through *base.
__device__ __forceinline__ int64_t epi_index(const Epilogue& e, int m, int n, void** base) {
    switch (e.mode) {
        default:
        case EPI_PLAIN:
            *base = e.C;
            return (int64_t)m * e.ldc + n;
        case EPI_ROWPTR: {
            int b = m / e.rows_per_batch, r = m - b * e.rows_per_batch;
            *base = e.batch_ptrs[b];
            return (int64_t)r * e.ldc + n;
        }
        case EPI_XKV: {
            // n -> (layer, kv, head, e);  m -> (batch b, frame r), or through the row maps when they are given
            int b = m / e.rows_per_batch, r = m - b * e.rows_per_batch;
            if (e.row_slot) { b = e.row_slot[m]; r = e.row_pos[m]; }
            int two_d = 2 * e.d_model;
            int l = n / two_d, rem = n - l * two_d;
            int kv = rem / e.d_model, c = rem - kv * e.d_model;
            int h = c >> 6, el = c & 63;
            *base = e.batch_ptrs[b];
            return ((((int64_t)l * 2 + kv) * e.n_head + h) * e.kv_len + r) * 64 + el;
        }
        case EPI_SELF_QKV: {
            int part = n / e.d_model, c = n - part * e.d_model;
            if (part == 0) {                       // q: plain [rows, d_model]
                *base = e.C;
                return (int64_t)m * e.ldc + c;
            }
            int h = c >> 6, el = c & 63;
            *base = e.batch_ptrs[e.row_slot[m]];
            return ((((int64_t)e.layer * 2 + (part - 1)) * e.n_head + h) * e.kv_len + e.row_pos[m]) * 64 + el;
        }
    }
}

__device__ __forceinline__ bool epi_row_dropped(const Epilogue& e, int m) {
    return e.mode == EPI_ROWPTR && (m % e.rows_per_batch) >= e.rows_valid;
}

__device__ __forceinline__ void epi_store1(const Epilogue& e, int m, int n, float acc) {
    if (epi_row_dropped(e, m)) return;
    float v = epi_math(e, acc, m, n);
    void* base;
    int64_t idx = epi_index(e, m, n, &base);
    if (e.c_type == DT_F32) reinterpret_cast<float*>(base)[idx] = v;
    else reinterpret_cast<bf16*>(base)[idx] = __float2bfloat16_rn(v);
}

// 8 consecutive columns n0..n0+7 (n0 % 8 == 0, all < N, same head): vector stores.
__device__ __forceinline__ void epi_store8(const Epilogue& e, int m, int n0, const float* acc) {
    if (epi_row_dropped(e, m)) return;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = epi_math(e, acc[j], m, n0 + j);
    void* base;
    int64_t idx = epi_index(e, m, n0, &base);
    if (e.c_type == DT_F32) {
        float* p = reinterpret_cast<float*>(base) + idx;
        if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
            reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
            reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) p[j] = v[j];
        }
    } else {
        bf16* p = reinterpret_cast<bf16*>(base) + idx;
        if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
            __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]);
            __nv_bfloat162 h1 = __floats2bfloat162_rn(v[2], v[3]);
            __nv_bfloat162 h2 = __floats2bfloat162_rn(v[4], v[5]);
            __nv_bfloat162 h3 = __floats2bfloat162_rn(v[6], v[7]);
            uint4 u;
            u.x = *reinterpret_cast<uint32_t*>(&h0);
            u.y = *reinterpret_cast<uint32_t*>(&h1);
            u.z = *reinterpret_cast<uint32_t*>(&h2);
            u.w = *reinterpret_cast<uint32_t*>(&h3);
            *reinterpret_cast<uint4*>(p) = u;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) p[j] = __float2bfloat16_rn(v[j]);
        }
    }
}

// ---------------------------------------------------------------------------------
// Factored destination addressing for the tensor-core GEMM epilogue:
//   address(m, n) = rowptr(m, variant) + colterm(n) * elem_size,  variant chosen per 8-column chunk.
// rowptr is computed once per tile and row (it hides the per-batch base pointer and every div/mod on m),
// colterm once per chunk and lane, so the per-element work is an add.
// ---------------------------------------------------------------------------------
struct EpiRow {
    char* ptr0;           // destination row base for variant 0 (nullptr: row is not stored)
    char* ptr1;           // variant 1 (EPI_SELF_QKV k/v planes); unused otherwise
    const float* res;     // residual row (already offset to column 0) or nullptr
};

__device__ __forceinline__ EpiRow epi_row(const Epilogue& e, int m, int M) {
    EpiRow r{nullptr, nullptr, nullptr};
    if (m >= M) return r;
    const int es = (e.c_type == DT_F32) ? 4 : 2;
    switch (e.mode) {
        default:
        case EPI_PLAIN:
            r.ptr0 = reinterpret_cast<char*>(e.C) + (int64_t)m * e.ldc * es;
            if (e.residual) r.res = e.residual + (int64_t)m * e.ldr;
            break;
        case EPI_ROWPTR: {
            int b = m / e.rows_per_batch, rr = m - b * e.rows_per_batch;
            if (rr < e.rows_valid) {
                r.ptr0 = reinterpret_cast<char*>(e.batch_ptrs[b]) + (int64_t)rr * e.ldc * es;
                if (e.residual) r.res = e.residual + (int64_t)rr * e.ldr;
            }
            break;
        }
        case EPI_XKV: {
            int b = m / e.rows_per_batch, rr = m - b * e.rows_per_batch;
            if (e.row_slot) { b = e.row_slot[m]; rr = e.row_pos[m]; }     // incremental encoder: row -> (session, ring slot)
            r.ptr0 = reinterpret_cast<char*>(e.batch_ptrs[b]) + (int64_t)rr * 64 * es;
            break;
        }
        case EPI_SELF_QKV:
            r.ptr0 = reinterpret_cast<char*>(e.C) + (int64_t)m * e.ldc * es;
            r.ptr1 = reinterpret_cast<char*>(e.batch_ptrs[e.row_slot[m]]) + (int64_t)e.row_pos[m] * 64 * es;
            break;
    }
    return r;
}

// element offset of column n (and which row-pointer variant its chunk uses)
__device__ __forceinline__ int64_t epi_col(const Epilogue& e, int n, int* variant) {
    *variant = 0;
    switch (e.mode) {
        default:
        case EPI_PLAIN:
        case EPI_ROWPTR:
            return n;
        case EPI_XKV: {
            int two_d = 2 * e.d_model;
            int l = n / two_d, rem = n - l * two_d;
            int kv = rem / e.d_model, c = rem - kv * e.d_model;
            return (((int64_t)l * 2 + kv) * e.n_head + (c >> 6)) * e.kv_len * 64 + (c & 63);
        }
        case EPI_SELF_QKV: {
            int part = n / e.d_model, c = n - part * e.d_model;
            if (part == 0) return c;
            *variant = 1;
            return (((int64_t)e.layer * 2 + (part - 1)) * e.n_head + (c >> 6)) * e.kv_len * 64 + (c & 63);
        }
    }
}

#endif  // __CUDACC__

}  // namespace wlk
