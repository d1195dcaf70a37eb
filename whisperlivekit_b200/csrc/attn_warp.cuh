// One warp per query row of head width 64, written once for the Whisper decoder's self-attention, the causal Qwen3
// tower and the windowed tower's fp32 mode.  The kernels keep their grid mapping, job decoding and loop over queries;
// key addressing comes in as callables.
#pragma once
#include "common.cuh"

namespace wlk {

template <typename T> struct RowVec;          // 16-byte slice of a 64-wide K/V row held by one lane
template <> struct RowVec<bf16> {
    static constexpr int N = 8;
    typedef uint4 Raw;
    static __device__ __forceinline__ Raw load(const bf16* p) { return *reinterpret_cast<const uint4*>(p); }
    static __device__ __forceinline__ void unpack(const Raw& u, float* o) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) { o[2 * i] = __low2float(h[i]); o[2 * i + 1] = __high2float(h[i]); }
    }
};
template <> struct RowVec<float> {
    static constexpr int N = 4;
    typedef float4 Raw;
    static __device__ __forceinline__ Raw load(const float* p) { return *reinterpret_cast<const float4*>(p); }
    static __device__ __forceinline__ void unpack(const Raw& v, float* o) { o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w; }
};

// softmax(q k^T) v of one query row over keys 0 .. n_keys - 1 (n_keys <= 32 * MAXK), called by a whole warp.  qs is the
// row in shared memory (64 floats, already scaled); k_row(key) / v_row(key) return the key's 64-wide K / V row, 16-byte
// aligned; out is the 64-wide output row.  Lanes own keys lane, lane + 32, ... for the scores (whole K rows per lane,
// 128-bit loads), the softmax runs on warp shuffles, then lanes own two output columns each and walk the keys with the
// probabilities broadcast by shuffle.  Only keys below n_keys are read.
template <typename T, int MAXK, typename KRow, typename VRow>
__device__ __forceinline__ void attend_row_warp(const float* qs, int n_keys, KRow k_row, VRow v_row, T* out) {
    constexpr int VN = RowVec<T>::N;
    const int lane = threadIdx.x & 31;
    float sc[MAXK];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < MAXK; ++i) {
        const int key = lane + 32 * i;
        float a = -INFINITY;
        if (key < n_keys) {
            a = 0.f;
            const T* kr = k_row(key);
#pragma unroll
            for (int c = 0; c < 64 / VN; ++c) {
                float kv[VN];
                RowVec<T>::unpack(RowVec<T>::load(kr + c * VN), kv);
#pragma unroll
                for (int j = 0; j < VN; ++j) a = fmaf(qs[c * VN + j], kv[j], a);
            }
        }
        sc[i] = a;
        mx = fmaxf(mx, a);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < MAXK; ++i) {
        const float p = (lane + 32 * i < n_keys) ? expf(sc[i] - mx) : 0.f;
        sc[i] = p;
        sum += p;
    }
    sum = warp_sum(sum);
    float o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int i = 0; i < MAXK; ++i) {
        if (32 * i >= n_keys) break;                   // warp-uniform
        const int lim = min(32, n_keys - 32 * i);
        // 16 V rows are fetched before any is used: a serial walk would expose one global-load latency per key
        for (int l0 = 0; l0 < lim; l0 += 16) {
            float v0[16], v1[16];
#pragma unroll
            for (int u = 0; u < 16; ++u) {
                const T* vr = v_row(32 * i + min(l0 + u, lim - 1)) + 2 * lane;
                v0[u] = to_f32(vr[0]);
                v1[u] = to_f32(vr[1]);
            }
#pragma unroll
            for (int u = 0; u < 16; ++u) {
                const float p = (l0 + u < lim) ? __shfl_sync(0xffffffffu, sc[i], (l0 + u) & 31) : 0.f;
                o0 = fmaf(p, v0[u], o0);
                o1 = fmaf(p, v1[u], o1);
            }
        }
    }
    const float inv = 1.0f / sum;
    out[2 * lane] = from_f32<T>(o0 * inv);
    out[2 * lane + 1] = from_f32<T>(o1 * inv);
}

}  // namespace wlk
