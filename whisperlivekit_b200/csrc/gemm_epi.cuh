// Epilogue and tile rasterisation of the wgmma GEMM kernel.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace wlk {

// erf-GELU for the tensor-core epilogue.  erf by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far below
// the bf16 rounding of everything this epilogue feeds): 5 FMAs, one MUFU.RCP and one MUFU.EX2 instead of
// the ~35-instruction erff(): the warpgroup's tensor pipe idles while its epilogue runs.
__device__ __forceinline__ float gelu_erf_fast(float x) {
    const float z = fabsf(x) * 0.70710678118654752440f;
    const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
    float p = fmaf(1.061405429f, t, -1.453152027f);
    p = fmaf(p, t, 1.421413741f);
    p = fmaf(p, t, -0.284496736f);
    p = fmaf(p, t, 0.254829592f);
    p *= t;
    const float e = 1.0f - p * __expf(-z * z);        // erf(|x| / sqrt 2)
    return 0.5f * x * (1.0f + copysignf(e, x));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// Fused epilogue of one warpgroup's 64 x BN accumulator, straight from the wgmma fragment: a thread owns, for every
// 8-column chunk, two adjacent columns of rows g and g + 8 (ptx.cuh), so the four lanes of a quad write one 32-byte
// (fp32) or 16-byte (bf16) run of a row.  The rows' destination pointers -- including every div/mod of the scatter
// modes -- are computed once per tile (`row`), the column part once per chunk (epi_col; a chunk never straddles a head).
template <int BN>
__device__ __forceinline__ void epilogue_fragment_tile(const Epilogue& epi, const EpiRow (&row)[2], float (&acc)[BN / 2],
                                                       int n_tile_base, int N, int lane) {
    const int es = (epi.c_type == DT_F32) ? 4 : 2;
    const int t2 = 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
        const int n0 = n_tile_base + c * 8;
        if (n0 >= N) break;
        int variant;
        const int64_t coff = (epi_col(epi, n0, &variant) + t2) * es;
        const int n = n0 + t2;
        const bool ok0 = n < N, ok1 = n + 1 < N;
        float b0 = 0.f, b1 = 0.f;
        if (epi.bias) { if (ok0) b0 = __ldg(epi.bias + n); if (ok1) b1 = __ldg(epi.bias + n + 1); }
        const bool scaled = (epi.scale_period ? (n0 % epi.scale_period) : n0) < epi.scale_cols;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            char* p = variant ? row[h].ptr1 : row[h].ptr0;
            if (p == nullptr || !ok0) continue;
            p += coff;
            float v0 = acc[4 * c + 2 * h] + b0, v1 = acc[4 * c + 2 * h + 1] + b1;
            if (epi.gelu == 1) { v0 = gelu_erf_fast(v0); v1 = gelu_erf_fast(v1); }
            else if (epi.gelu == 2) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            else if (epi.gelu == 3) { v0 = __fdividef(v0, 1.0f + __expf(-v0)); v1 = __fdividef(v1, 1.0f + __expf(-v1)); }
            if (scaled) { v0 *= epi.col_scale; v1 *= epi.col_scale; }
            if (row[h].res) {
                v0 += row[h].res[n];
                if (ok1) v1 += row[h].res[n + 1];
            }
            if (es == 4) {
                if (ok1 && (reinterpret_cast<uintptr_t>(p) & 7) == 0) *reinterpret_cast<float2*>(p) = make_float2(v0, v1);
                else { reinterpret_cast<float*>(p)[0] = v0; if (ok1) reinterpret_cast<float*>(p)[1] = v1; }
            } else {
                if (ok1 && (reinterpret_cast<uintptr_t>(p) & 3) == 0) *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(v0, v1);
                else { reinterpret_cast<bf16*>(p)[0] = __float2bfloat16_rn(v0); if (ok1) reinterpret_cast<bf16*>(p)[1] = __float2bfloat16_rn(v1); }
            }
        }
    }
}

// Tile rasterisation shared by the producer and the consumer warps.  Work item t -> (m block, n block): tiles are walked
// in bands of `band` m-blocks, n-blocks fastest-but-one inside a band, so the ~num_sms tiles in flight at
// any time cover one band x a few n-blocks: the band's A rows are fetched from HBM once and then served
// from L2 for the whole sweep over n, and the few W panels in flight are shared by every CTA.
__device__ __forceinline__ void tile_coords(int t, int num_m, int num_n, int band, int* m_blk, int* n_blk) {
    const int per_band = band * num_n;
    const int b = t / per_band;
    const int r = t - b * per_band;
    const int h = min(band, num_m - b * band);       // height of this (possibly last, shorter) band
    *n_blk = r / h;
    *m_blk = b * band + (r - (*n_blk) * h);
}

// Pull the fp32 residual values a row's epilogue will add (`n_cols` columns from n_begin) into L2 while the tile's
// MMAs are still running, so the epilogue's residual loads are L2 hits instead of HBM round trips.
__device__ __forceinline__ void epilogue_prefetch_residual(const EpiRow& row, int n_begin, int n_cols, int N) {
    if (row.res == nullptr) return;
    const char* p = reinterpret_cast<const char*>(row.res + n_begin);
    const int bytes = min(n_cols, max(0, N - n_begin)) * 4;
    for (int off = 0; off < bytes; off += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + off));
}

// split-K: this K range's raw accumulators to / from a [BM][BN] fp32 tile of the global scratch (`tile_row0` points at
// the warpgroup's first row of that tile); same fragment positions both ways
template <int BN>
__device__ __forceinline__ void partials_store(float* tile_row0, const float (&acc)[BN / 2], int warp_in_wg, int lane) {
    float* r0 = tile_row0 + (int64_t)(warp_in_wg * 16 + (lane >> 2)) * BN + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
        __stcg(reinterpret_cast<float2*>(r0 + c * 8), make_float2(acc[4 * c], acc[4 * c + 1]));
        __stcg(reinterpret_cast<float2*>(r0 + 8 * BN + c * 8), make_float2(acc[4 * c + 2], acc[4 * c + 3]));
    }
}
template <int BN>
__device__ __forceinline__ void partials_add(const float* tile_row0, float (&acc)[BN / 2], int warp_in_wg, int lane) {
    const float* r0 = tile_row0 + (int64_t)(warp_in_wg * 16 + (lane >> 2)) * BN + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
        const float2 a = __ldcg(reinterpret_cast<const float2*>(r0 + c * 8));
        const float2 b = __ldcg(reinterpret_cast<const float2*>(r0 + 8 * BN + c * 8));
        acc[4 * c] += a.x; acc[4 * c + 1] += a.y; acc[4 * c + 2] += b.x; acc[4 * c + 3] += b.y;
    }
}

bool make_tmap_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols, std::string* err);

}  // namespace wlk
