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
                if (ok1 && (reinterpret_cast<uintptr_t>(p) & 3) == 0) *reinterpret_cast<uint32_t*>(p) = ptx::pack_bf16x2(v0, v1);
                else { reinterpret_cast<bf16*>(p)[0] = __float2bfloat16_rn(v0); if (ok1) reinterpret_cast<bf16*>(p)[1] = __float2bfloat16_rn(v1); }
            }
        }
    }
}

// Fused epilogue of a ping-pong consumer's whole 128 x 128 tile.  acc[h] is the m64n128 fragment of tile rows 64h..64h+63,
// row0 the thread's first row (tile row 16 wq + g), so that it owns rows row0 + 64h + 8r (fragment positions as in ptx.cuh).  It runs while
// the other consumer's MMAs keep the tensor pipe busy, so it is kept short and straight: every per-tile decision
// (activation, column scale, residual, output type) is taken once outside the element loops, the arithmetic runs in
// registers, every residual value is loaded before the first store (C may alias the residual: x += A W^T in place, so a
// load behind a store would wait for it), and loads and stores are global-space.
template <bool F32>
__device__ __forceinline__ void epilogue_store_tile128(const Epilogue& epi, const EpiRow (&row)[4], const float (&acc)[2][64],
                                                       int n_base, int N, int lane) {
    constexpr int es = F32 ? 4 : 2;
    const int t2 = 2 * (lane & 3);
    // a chunk's column offset is even, so a row whose base is aligned takes a two-element store at every chunk
    bool vec = n_base + 128 <= N;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        vec = vec && row[i].ptr0 != nullptr && (reinterpret_cast<uintptr_t>(row[i].ptr0) & (2 * es - 1)) == 0;
        if (epi.mode == EPI_SELF_QKV)
            vec = vec && row[i].ptr1 != nullptr && (reinterpret_cast<uintptr_t>(row[i].ptr1) & (2 * es - 1)) == 0;
    }
    if (vec) {                                               // whole tile, aligned rows: straight-line stores
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            int variant;
            const int64_t coff = (epi_col(epi, n_base + c * 8, &variant) + t2) * es;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                char* p = (variant ? row[i].ptr1 : row[i].ptr0) + coff;
                const float v0 = acc[i >> 1][4 * c + 2 * (i & 1)], v1 = acc[i >> 1][4 * c + 2 * (i & 1) + 1];
                if (F32) ptx::st_global_f32x2(p, v0, v1);
                else ptx::st_global_b32(p, ptx::pack_bf16x2(v0, v1));
            }
        }
        return;
    }
    // tail tiles (rows past M, dropped rows, a partial column block) and unaligned rows
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        const int n0 = n_base + c * 8;
        if (n0 >= N) break;
        int variant;
        const int64_t coff = (epi_col(epi, n0, &variant) + t2) * es;
        const int n = n0 + t2;
        const bool ok0 = n < N, ok1 = n + 1 < N;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            char* p = variant ? row[i].ptr1 : row[i].ptr0;
            if (p == nullptr || !ok0) continue;
            p += coff;
            const float v0 = acc[i >> 1][4 * c + 2 * (i & 1)], v1 = acc[i >> 1][4 * c + 2 * (i & 1) + 1];
            if (F32) {
                if (ok1 && (reinterpret_cast<uintptr_t>(p) & 7) == 0) ptx::st_global_f32x2(p, v0, v1);
                else { ptx::st_global_f32(p, v0); if (ok1) ptx::st_global_f32(p + 4, v1); }
            } else {
                if (ok1 && (reinterpret_cast<uintptr_t>(p) & 3) == 0) ptx::st_global_b32(p, ptx::pack_bf16x2(v0, v1));
                else {
                    ptx::st_global_b16(p, __bfloat16_as_ushort(__float2bfloat16_rn(v0)));
                    if (ok1) ptx::st_global_b16(p + 2, __bfloat16_as_ushort(__float2bfloat16_rn(v1)));
                }
            }
        }
    }
}

template <typename F>
__device__ __forceinline__ void epilogue_map_tile128(float (&acc)[2][64], F f) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[h][j] = f(acc[h][j]);
}

// bias, activation, column scale of a ping-pong consumer's 128 x 128 tile: registers only.  FP8 (e4m3 operands): first
// acc[m, n] * a_scale[m] * w_scale[n], a row scale at a time and then the column scales by shuffle, so that no more than
// a few loaded scales are live next to the 128 accumulators.
template <bool FP8 = false>
__device__ __forceinline__ void epilogue_math_tile128(const Epilogue& epi, float (&acc)[2][64], int n_base, int N, int lane,
                                                      int row0 = 0, int M = 0) {
    const int t2 = 2 * (lane & 3);
    if (FP8) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = row0 + 8 * (i & 1) + 64 * (i >> 1);
            const float sa = m < M ? __ldg(epi.a_scale + m) : 0.f;
#pragma unroll
            for (int c = 0; c < 16; ++c) { acc[i >> 1][4 * c + 2 * (i & 1)] *= sa; acc[i >> 1][4 * c + 2 * (i & 1) + 1] *= sa; }
        }
        // column scales: lane l loads columns 4l .. 4l + 3 of the tile once; a chunk's pair comes by shuffle (loading all
        // 32 of a thread's scales next to the bias would hold 64 loaded values beside the 128 accumulators)
        float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
        {
            const int n = n_base + 4 * lane;
            if (n + 3 < N && (reinterpret_cast<uintptr_t>(epi.w_scale + n) & 15) == 0) wv = __ldg(reinterpret_cast<const float4*>(epi.w_scale + n));
            else {
                if (n < N) wv.x = __ldg(epi.w_scale + n);
                if (n + 1 < N) wv.y = __ldg(epi.w_scale + n + 1);
                if (n + 2 < N) wv.z = __ldg(epi.w_scale + n + 2);
                if (n + 3 < N) wv.w = __ldg(epi.w_scale + n + 3);
            }
        }
        const bool odd = (lane & 1) != 0;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            const int src = 2 * c + ((lane & 3) >> 1);       // the lane holding columns 8c + 2t, +1
            const float x = __shfl_sync(0xffffffffu, wv.x, src), y = __shfl_sync(0xffffffffu, wv.y, src);
            const float z = __shfl_sync(0xffffffffu, wv.z, src), w = __shfl_sync(0xffffffffu, wv.w, src);
            const float w0 = odd ? z : x, w1 = odd ? w : y;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                acc[h][4 * c] *= w0; acc[h][4 * c + 1] *= w1; acc[h][4 * c + 2] *= w0; acc[h][4 * c + 3] *= w1;
            }
        }
    }
    if (epi.bias) {
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            const int n = n_base + 8 * c + t2;
            const float b0 = n < N ? __ldg(epi.bias + n) : 0.f, b1 = n + 1 < N ? __ldg(epi.bias + n + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                acc[h][4 * c] += b0; acc[h][4 * c + 1] += b1; acc[h][4 * c + 2] += b0; acc[h][4 * c + 3] += b1;
            }
        }
    }
    switch (epi.gelu) {
        case 1: epilogue_map_tile128(acc, [](float v) { return gelu_erf_fast(v); }); break;
        case 2: epilogue_map_tile128(acc, [](float v) { return fmaxf(v, 0.f); }); break;
        case 3: epilogue_map_tile128(acc, [](float v) { return __fdividef(v, 1.0f + __expf(-v)); }); break;
        default: break;
    }
    if (epi.scale_cols > 0) {
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            const int n0 = n_base + 8 * c;
            if ((epi.scale_period ? (n0 % epi.scale_period) : n0) >= epi.scale_cols) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[h][4 * c + j] *= epi.col_scale;
        }
    }
}

// e4m3 output: every row divided by its scale c_scale[m] (a zero scale stores zeros), ready for the saturating convert
__device__ __forceinline__ void epilogue_out_scale_tile128(const Epilogue& epi, int row0, int M, float (&acc)[2][64]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = row0 + 8 * (i & 1) + 64 * (i >> 1);
        const float s = m < M ? __ldg(epi.c_scale + m) : 0.f;
        const float inv = s > 0.f ? 1.0f / s : 0.f;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            acc[i >> 1][4 * c + 2 * (i & 1)] *= inv;
            acc[i >> 1][4 * c + 2 * (i & 1) + 1] *= inv;
        }
    }
}

// The register-path epilogue of a whole tile (the scatter modes, and plain outputs whose pitch or base a tensor map
// cannot address): residual from global memory, stores straight from the fragment.  FP8: e4m3 operands (an e4m3 output
// always leaves through the staged epilogue: gemm_tcgen05_supported).
template <bool FP8 = false>
__device__ __forceinline__ void epilogue_tile128(const Epilogue& epi, int row0, int M, float (&acc)[2][64], int n_base, int N,
                                                 int lane) {
    const int t2 = 2 * (lane & 3);
    const bool full = n_base + 128 <= N;
    epilogue_math_tile128<FP8>(epi, acc, n_base, N, lane, row0, M);
    if (epi.residual) {
        // each pass derives the row pointers it needs: none of them stays live next to the 128 accumulators
        EpiRow row[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) row[i] = epi_row(epi, row0 + 8 * (i & 1) + 64 * (i >> 1), M);
        bool vec = full;
#pragma unroll
        for (int i = 0; i < 4; ++i) vec = vec && row[i].res != nullptr && (reinterpret_cast<uintptr_t>(row[i].res) & 7) == 0;
        if (vec) {
            // the whole tile in one basic block: the scheduler batches the 64 loads as far as registers allow
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < 16; ++c) {
                    const float2 v = ptx::ld_global_f32x2(row[i].res + n_base + 8 * c + t2);
                    acc[i >> 1][4 * c + 2 * (i & 1)] += v.x;
                    acc[i >> 1][4 * c + 2 * (i & 1) + 1] += v.y;
                }
        } else {
            // tail tiles (rows past M, dropped rows, a partial column block) and unaligned rows
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float* res = row[i].res;
                if (res == nullptr) continue;
#pragma unroll
                for (int c = 0; c < 16; ++c) {
                    const int n = n_base + 8 * c + t2;
                    if (n < N) acc[i >> 1][4 * c + 2 * (i & 1)] += ptx::ld_global_f32(res + n);
                    if (n + 1 < N) acc[i >> 1][4 * c + 2 * (i & 1) + 1] += ptx::ld_global_f32(res + n + 1);
                }
            }
        }
    }
    EpiRow row[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) row[i] = epi_row(epi, row0 + 8 * (i & 1) + 64 * (i >> 1), M);
    if (epi.c_type == DT_F32) epilogue_store_tile128<true>(epi, row, acc, n_base, N, lane);
    else epilogue_store_tile128<false>(epi, row, acc, n_base, N, lane);
}

// Staged epilogue of a ping-pong consumer's 128 x 128 tile into a plain row-major C (bias, activation and column scale
// already applied, no residual).  The tile leaves in NS sub-tiles of 128 rows x 128 bytes (32 fp32, 64 bf16 or 128 e4m3
// columns) through the consumer's two 16 KiB buffers at `buf`, which hold them 128B-swizzled as the tensor map tmC expects:
// 16-byte unit u of row r sits at unit u ^ (r & 7), so every warp-wide fragment store touches each bank once per 128
// bytes.  One thread (the warpgroup's first) stores a written buffer by TMA while the warpgroup writes the other; a
// buffer is rewritten once its previous store has read it.  TMA clips rows past M and columns past N.  The values are
// those epilogue_tile128 stores.  ES: bytes per element of C.
template <int ES>
__device__ __forceinline__ void epilogue_tma_tile128(const float (&acc)[2][64], const CUtensorMap* tmC, int m_base,
                                                     int n_base, uint32_t buf, int epi_bar, int wq, int lane) {
    constexpr bool F32 = ES == 4;
    constexpr int NS = ES == 4 ? 4 : ES == 2 ? 2 : 1;  // sub-tiles per tile
    constexpr int CPS = 16 / NS;                       // 8-column chunks per sub-tile
    const int g = lane >> 2, t = lane & 3;
    const bool leader = wq == 0 && lane == 0;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
        const uint32_t b = buf + (s & 1) * (128 * 128);
        if (leader) ptx::bulk_wait_group_read<1>();    // the store that last read buffer b (two sub-tiles ago) is done
        ptx::named_bar_sync<128>(epi_bar);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t row = b + (16 * wq + g + 8 * (i & 1) + 64 * (i >> 1)) * 128;   // (row & 7) == g
#pragma unroll
            for (int cl = 0; cl < CPS; ++cl) {
                const int j = 4 * (s * CPS + cl) + 2 * (i & 1);
                if (F32) ptx::st_shared_f32x2(row + (((2 * cl + (t >> 1)) ^ g) << 4) + 8 * (t & 1), acc[i >> 1][j], acc[i >> 1][j + 1]);
                else if (ES == 1) ptx::st_shared_b16(row + (((cl >> 1) ^ g) << 4) + 8 * (cl & 1) + 2 * t,
                                                     ptx::pack_e4m3x2(acc[i >> 1][j], acc[i >> 1][j + 1]));
                else ptx::st_shared_b32(row + ((cl ^ g) << 4) + 4 * t, ptx::pack_bf16x2(acc[i >> 1][j], acc[i >> 1][j + 1]));
            }
        }
        ptx::fence_proxy_async_smem();                 // the writes above, before the async proxy reads the buffer
        ptx::named_bar_sync<128>(epi_bar);
        if (leader) {
            ptx::tma_store_2d(tmC, b, n_base + s * (128 / NS), m_base);
            ptx::bulk_commit_group();
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
