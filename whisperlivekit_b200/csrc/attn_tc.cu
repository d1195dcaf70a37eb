// Fused attention on the Hopper tensor cores (sm_90a, wgmma).
//   O = softmax(Q K^T) V over all 1500 positions, no mask (reference whisper/model.py:148-173);
//   q and k arrive pre-scaled by d_head^-0.25 from the QKV GEMM epilogue.
//
// One CTA per (128-query tile, head, stream):
//   warps 0-7  two warpgroups, 64 query rows each.  Per 128-key tile: S = Q K^T (wgmma, both operands in shared
//              memory, M64 N128 K16 x4) lands in registers; online softmax on the fragment (a row lives in the
//              four lanes of a quad: running maximum and sum, O rescaled in registers when the maximum moves);
//              P is packed to bf16 in place -- the accumulator fragment of S is the A fragment of the next MMA --
//              and O += P V runs with P from registers and V MN-major from shared memory (M64 N64 K16 x8).
//              The two warpgroups drift apart by themselves, so one's exponentials overlap the other's MMAs.
//   warp 8     TMA producer: Q tile once, then 128-key K and V tiles (128B-swizzled) through a 2-stage
//              mbarrier ring, straight out of the fused [rows, 3d] qkv buffer
#include <cudaTypedefs.h>

#include "kernels.cuh"
#include "ptx.cuh"

namespace wlk {

bool make_tmap_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols, std::string* err);

namespace {

constexpr int BQ = 128, BKV = 128, DH = 64;
constexpr int ATT_MMA_WARPS = 8;
constexpr int ATT_THREADS = 32 * ATT_MMA_WARPS + 32;  // two softmax/MMA warpgroups, then the TMA warp
constexpr uint32_t TILE_BYTES = BQ * DH * 2;          // 16 KB: Q, K and V tiles all are 128 x 64 bf16
// Shared-memory layout.  X3 (WLK_PREC_BF16X3): every operand is two bf16 planes (hi, lo); Q K^T and P V are each
// three MMAs (hi hi + lo hi + hi lo) into the same fp32 accumulator, P is split like the other operands, the output is
// fp32.
template <bool X3> struct AttLayout {
    static constexpr uint32_t NP = X3 ? 2 : 1;                               // planes per operand
    static constexpr uint32_t SM_Q = 0;                                      // [NP] tiles
    static constexpr uint32_t SM_K = NP * TILE_BYTES;                        // [2 stages][NP]
    static constexpr uint32_t SM_V = SM_K + 2 * NP * TILE_BYTES;             // [2 stages][NP]
    static constexpr uint32_t SM_BAR = SM_V + 2 * NP * TILE_BYTES;
    static constexpr uint32_t SMEM = SM_BAR + 64 + 1024;
};
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ float fast_exp2(float x) {      // MUFU.EX2, flush-to-zero, exp2(-inf) = 0
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// MODE 0: encoder self-attention, Q/K/V tiles all come out of the fused qkv buffer (tensor map `tm`).
// MODE 1: decoder cross-attention of a prefill (many query rows per session): Q tiles from the packed
//         query buffer (`tm`), K/V tiles from the session's head-major cross-K/V planes through a
//         per-session tensor map kept in global memory (`kv_maps[job.slot]`).  Alignment heads are
//         skipped here: their rows need the exactly normalised probabilities exported, which the
//         SIMT kernel produces.
// MODE 2: decoder SELF-attention of a prefill, causal: Q as in mode 1, K/V tiles from the session's self-K/V
//         cache planes [L][2][H][n_text_ctx][64] (per-session tensor map); query row at position p sees keys
//         0..p -- the mask is applied per row where the probabilities are formed (masked keys get exactly 0),
//         and only the key tiles up to the tile's last position are visited.  A long context prefix (the
//         reference keeps up to n_text_ctx - 20 = 428 tokens, align_att_base.py:100-113) is tens of thousands of
//         query rows x 32 layers per tick, far too many for the SIMT kernel.
constexpr int MODE_ENC = 0, MODE_CROSS = 1, MODE_SELF = 2;
template <int MODE, bool X3>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tm_lo,
               const CUtensorMap* __restrict__ kv_maps,
               const DecJob* __restrict__ jobs, int layer, const int32_t* __restrict__ align_rank,
               int n_head, int d_model, int kv_len, void* __restrict__ out_ptr) {
    constexpr bool CROSS = MODE != MODE_ENC;              // Q from the packed query buffer, K/V through a per-session map
    static_assert(!(CROSS && X3), "the split-operand variant serves the encoder only");
    using AL = AttLayout<X3>;
    constexpr uint32_t SM_Q = AL::SM_Q, SM_K = AL::SM_K, SM_V = AL::SM_V, SM_BAR = AL::SM_BAR, NP = AL::NP;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t sbase = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_q = sbase + SM_BAR;
    const uint32_t bar_kv_full = bar_q + 8;       // [2]
    const uint32_t bar_kv_empty = bar_q + 24;     // [2]

    ptx::griddep_launch();                   // programmatic dependent launch: see launch_pdl (common.cuh)
    ptx::griddep_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
    int NT = (N_CTX + BKV - 1) / BKV;                    // 12 key tiles (encoder, cross)
    int pos0 = 0;                                        // MODE_SELF: position of the tile's first query row
    // tile origins (tensor-map coordinates) and the number of query rows this CTA owns
    const CUtensorMap* tm_kv = &tm;
    int q_row, q_col = h * DH, k_row, k_col, v_row, v_col, out_row, n_q;
    if constexpr (CROSS) {
        const DecJob job = jobs[b];
        if (q0 >= job.n_rows) return;                                            // uniform: before any barrier use
        if (MODE == MODE_CROSS && align_rank[layer * n_head + h] >= 0) return;
        tm_kv = kv_maps + job.slot;
        q_row = job.row_off + q0;
        k_row = (((layer * 2 + 0) * n_head) + h) * kv_len; k_col = 0;
        v_row = (((layer * 2 + 1) * n_head) + h) * kv_len; v_col = 0;
        out_row = job.row_off + q0;
        n_q = min(BQ, job.n_rows - q0);
        if (MODE == MODE_SELF) {
            pos0 = job.offset + q0;
            NT = (pos0 + n_q + BKV - 1) / BKV;                                   // keys 0 .. position of the last row
        }
    } else {
        q_row = b * N_CTX + q0;
        k_row = b * N_CTX; k_col = d_model + h * DH;
        v_row = b * N_CTX; v_col = 2 * d_model + h * DH;
        out_row = b * N_CTX + q0;
        n_q = min(BQ, N_CTX - q0);
    }

    if (warp == ATT_MMA_WARPS && lane == 0) {
        ptx::prefetch_tensormap(&tm);
        if (X3) ptx::prefetch_tensormap(&tm_lo);
        if (CROSS) ptx::prefetch_tensormap(tm_kv);
        ptx::mbar_init(bar_q, 1);
        for (int i = 0; i < 2; ++i) {
            ptx::mbar_init(bar_kv_full + 8 * i, 1);
            ptx::mbar_init(bar_kv_empty + 8 * i, ATT_MMA_WARPS);   // lane 0 of every MMA warp releases a stage
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == ATT_MMA_WARPS) {
        if (lane == 0) {
            ptx::mbar_arrive_expect_tx(bar_q, NP * TILE_BYTES);
            ptx::tma_load_2d(sbase + SM_Q, &tm, bar_q, q_col, q_row);
            if (X3) ptx::tma_load_2d(sbase + SM_Q + TILE_BYTES, &tm_lo, bar_q, q_col, q_row);
            for (int j = 0; j < NT; ++j) {
                const uint32_t s = j & 1, ph = (j >> 1) & 1;
                ptx::mbar_wait_mma(bar_kv_empty + 8 * s, ph ^ 1);
                ptx::mbar_arrive_expect_tx(bar_kv_full + 8 * s, 2 * NP * TILE_BYTES);
                ptx::tma_load_2d(sbase + SM_K + s * NP * TILE_BYTES, tm_kv, bar_kv_full + 8 * s, k_col, k_row + j * BKV);
                ptx::tma_load_2d(sbase + SM_V + s * NP * TILE_BYTES, tm_kv, bar_kv_full + 8 * s, v_col, v_row + j * BKV);
                if (X3) {
                    ptx::tma_load_2d(sbase + SM_K + (s * NP + 1) * TILE_BYTES, &tm_lo, bar_kv_full + 8 * s, k_col, k_row + j * BKV);
                    ptx::tma_load_2d(sbase + SM_V + (s * NP + 1) * TILE_BYTES, &tm_lo, bar_kv_full + 8 * s, v_col, v_row + j * BKV);
                }
            }
        }
        return;
    }

    // ---- softmax / MMA warpgroups.  Fragment geometry (ptx.cuh): this thread owns rows r0 and r0 + 8 of the query tile and,
    // in every 8-key chunk c of a key tile, keys 8c + 2t and 8c + 2t + 1; sc[4c + 2i + e] is (row r0 + 8i, key 8c + 2t + e).
    const int wg = warp >> 2, t2 = 2 * (lane & 3);
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    constexpr uint32_t WG_Q_OFF = 64 * DH * 2;            // the warpgroup's 64 rows of the Q tile
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // running row maximum (log2 domain) and this thread's share of the row sum
    ptx::mbar_wait_mma(bar_q, 0);
#pragma unroll 1
    for (int j = 0; j < NT; ++j) {
        const uint32_t s = j & 1;
        ptx::mbar_wait_mma(bar_kv_full + 8 * s, (j >> 1) & 1);
        float sc[64];
        {
            const uint64_t dq = ptx::wgmma_desc_sw128(sbase + SM_Q + wg * WG_Q_OFF);
            const uint64_t dk = ptx::wgmma_desc_sw128(sbase + SM_K + s * NP * TILE_BYTES);
            const uint64_t dql = ptx::wgmma_desc_sw128(sbase + SM_Q + TILE_BYTES + wg * WG_Q_OFF);
            const uint64_t dkl = ptx::wgmma_desc_sw128(sbase + SM_K + (s * NP + 1) * TILE_BYTES);
            ptx::wgmma_fence_regs(sc);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < DH / 16; ++k) {
                ptx::WgmmaSS<BKV>::mma(sc, dq + 2 * k, dk + 2 * k, k > 0 ? 1u : 0u);
                if (X3) {
                    ptx::WgmmaSS<BKV>::mma(sc, dql + 2 * k, dk + 2 * k, 1u);
                    ptx::WgmmaSS<BKV>::mma(sc, dq + 2 * k, dkl + 2 * k, 1u);
                }
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_regs(sc);
        }
        // keys past the end of the sequence (the last, 92-key tile) or -- causal -- past the row's own position score -inf
        if (MODE == MODE_SELF || j == NT - 1) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int n_valid = (MODE == MODE_SELF ? pos0 + r0 + 8 * i + 1 : N_CTX) - j * BKV;
#pragma unroll
                for (int c = 0; c < BKV / 8; ++c) {
                    if (c * 8 + t2 >= n_valid) sc[4 * c + 2 * i] = -INFINITY;
                    if (c * 8 + t2 + 1 >= n_valid) sc[4 * c + 2 * i + 1] = -INFINITY;
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float mx = -INFINITY;
#pragma unroll
            for (int c = 0; c < BKV / 8; ++c) mx = fmaxf(mx, fmaxf(sc[4 * c + 2 * i], sc[4 * c + 2 * i + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m[i], mx * LOG2E);
            const float m_ref = m_new == -INFINITY ? 0.f : m_new;     // a row with no visible key yet: every p is exp2(-inf) = 0
            const float alpha = fast_exp2(m[i] - m_ref);
            m[i] = m_new;
            if (alpha != 1.0f) {
                l[i] *= alpha;
#pragma unroll
                for (int c = 0; c < DH / 8; ++c) { o[4 * c + 2 * i] *= alpha; o[4 * c + 2 * i + 1] *= alpha; }
            }
            float rs = 0.f;
#pragma unroll
            for (int c = 0; c < BKV / 8; ++c) {
                const float p0 = fast_exp2(fmaf(sc[4 * c + 2 * i], LOG2E, -m_ref));
                const float p1 = fast_exp2(fmaf(sc[4 * c + 2 * i + 1], LOG2E, -m_ref));
                rs += p0 + p1;
                sc[4 * c + 2 * i] = p0; sc[4 * c + 2 * i + 1] = p1;
            }
            l[i] += rs;
        }
        // O += P V: the S fragment of keys 16k .. 16k + 15 is exactly the A fragment of the k-th K=16 step
        {
            const uint64_t dv = ptx::wgmma_desc_sw128(sbase + SM_V + s * NP * TILE_BYTES);
            const uint64_t dvl = ptx::wgmma_desc_sw128(sbase + SM_V + (s * NP + 1) * TILE_BYTES);
            uint32_t pa[BKV / 16][4];
            uint32_t pl[X3 ? BKV / 16 : 1][4];
#pragma unroll
            for (int k = 0; k < BKV / 16; ++k) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float p0 = sc[8 * k + 2 * e], p1 = sc[8 * k + 2 * e + 1];
                    const __nv_bfloat162 hb = __floats2bfloat162_rn(p0, p1);
                    pa[k][e] = *reinterpret_cast<const uint32_t*>(&hb);
                    if (X3) pl[k][e] = pack_bf16x2(p0 - __low2float(hb), p1 - __high2float(hb));   // P = hi + lo like every other operand
                }
            }
            ptx::wgmma_fence_regs(o);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BKV / 16; ++k) {           // 16 keys = 16 V rows of 128 B = 2048 B = +128 encoded
                ptx::wgmma_rs_n64_bt(o, pa[k], dv + 128 * k);
                if (X3) {
                    ptx::wgmma_rs_n64_bt(o, pl[k], dv + 128 * k);
                    ptx::wgmma_rs_n64_bt(o, pa[k], dvl + 128 * k);
                }
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_regs(o);
        }
        if (lane == 0) ptx::mbar_arrive(bar_kv_empty + 8 * s);      // this warp has read K and V of the stage
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        float ls = l[i];
        ls += __shfl_xor_sync(0xffffffffu, ls, 1);
        ls += __shfl_xor_sync(0xffffffffu, ls, 2);
        // (the IEEE division's slow path is a subroutine call; it is reachable only here, after the last
        // wgmma_wait<0>, where no wgmma group is in flight, so ptxas keeps the MMAs asynchronous)
        const float inv = 1.0f / ls;
        const int r = r0 + 8 * i;
        if (r >= n_q) continue;
        const int64_t off = (int64_t)(out_row + r) * d_model + h * DH + t2;
#pragma unroll
        for (int c = 0; c < DH / 8; ++c) {
            const float v0 = o[4 * c + 2 * i] * inv, v1 = o[4 * c + 2 * i + 1] * inv;
            if (X3) *reinterpret_cast<float2*>(reinterpret_cast<float*>(out_ptr) + off + c * 8) = make_float2(v0, v1);
            else *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(out_ptr) + off + c * 8) = pack_bf16x2(v0, v1);
        }
    }
}

}  // namespace

void enc_attention_tcgen05(const void* qkv, int batch, int n_head, int d_model, void* out, cudaStream_t st) {
    CUtensorMap tm;
    std::string err;
    WLK_CHECK(make_tmap_bf16_2d(&tm, qkv, (uint64_t)batch * N_CTX, (uint64_t)3 * d_model, (uint64_t)3 * d_model, BQ, DH, &err),
              "qkv tensor map: %s", err.c_str());
    static bool seen[64] = {};
    if (first_on_device(seen))
        CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel<MODE_ENC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AttLayout<false>::SMEM));
    dim3 grid((N_CTX + BQ - 1) / BQ, n_head, batch);
    attn_tc_kernel<MODE_ENC, false><<<grid, ATT_THREADS, AttLayout<false>::SMEM, st>>>(tm, tm, nullptr, nullptr, 0, nullptr, n_head, d_model, N_CTX, out);
    CUDA_CHECK(cudaGetLastError());
}

// WLK_PREC_BF16X3: qkv arrives as two bf16 planes [batch*1500, 3d] (hi, lo) -- the split of the fp32 QKV GEMM output --
// and the result is fp32 [batch*1500, d].
void enc_attention_tcgen05_x3(const void* qkv_hi, const void* qkv_lo, int batch, int n_head, int d_model, float* out, cudaStream_t st) {
    CUtensorMap tm, tml;
    std::string err;
    WLK_CHECK(make_tmap_bf16_2d(&tm, qkv_hi, (uint64_t)batch * N_CTX, (uint64_t)3 * d_model, (uint64_t)3 * d_model, BQ, DH, &err),
              "qkv tensor map: %s", err.c_str());
    WLK_CHECK(make_tmap_bf16_2d(&tml, qkv_lo, (uint64_t)batch * N_CTX, (uint64_t)3 * d_model, (uint64_t)3 * d_model, BQ, DH, &err),
              "qkv lo tensor map: %s", err.c_str());
    static bool seen[64] = {};
    if (first_on_device(seen))
        CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel<MODE_ENC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AttLayout<true>::SMEM));
    dim3 grid((N_CTX + BQ - 1) / BQ, n_head, batch);
    attn_tc_kernel<MODE_ENC, true><<<grid, ATT_THREADS, AttLayout<true>::SMEM, st>>>(tm, tml, nullptr, nullptr, 0, nullptr, n_head, d_model, N_CTX, out);
    CUDA_CHECK(cudaGetLastError());
}

// tensor map over one session's cross-K/V planes viewed as [L * 2 * H * 1500 rows, 64] bf16
void make_cross_kv_tmap(void* tmap_out_host, const void* cross_kv, int n_layer, int n_head) {
    std::string err;
    WLK_CHECK(make_tmap_bf16_2d(reinterpret_cast<CUtensorMap*>(tmap_out_host), cross_kv,
                                (uint64_t)n_layer * 2 * n_head * N_CTX, DH, DH, BKV, DH, &err),
              "cross-K/V tensor map: %s", err.c_str());
}

void dec_cross_attention_tcgen05(const void* q, int total_rows, const DecJob* jobs, int n_jobs, int max_rows, int layer,
                                 int n_head, int d_model, const void* kv_maps_dev, const int32_t* align_rank, void* out,
                                 cudaStream_t st) {
    CUtensorMap tm;
    std::string err;
    WLK_CHECK(make_tmap_bf16_2d(&tm, q, (uint64_t)total_rows, (uint64_t)d_model, (uint64_t)d_model, BQ, DH, &err),
              "query tensor map: %s", err.c_str());
    static bool seen[64] = {};
    if (first_on_device(seen))
        CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel<MODE_CROSS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AttLayout<false>::SMEM));
    dim3 grid((max_rows + BQ - 1) / BQ, n_head, n_jobs);
    CUDA_CHECK(launch_pdl(attn_tc_kernel<MODE_CROSS, false>, grid, dim3(ATT_THREADS), (size_t)AttLayout<false>::SMEM, st, tm, tm,
                          reinterpret_cast<const CUtensorMap*>(kv_maps_dev), jobs, layer, align_rank, n_head, d_model, N_CTX, out));
}

// tensor map over one session's self-K/V cache viewed as [L * 2 * H * n_text_ctx rows, 64] bf16
void make_self_kv_tmap(void* tmap_out_host, const void* self_kv, int n_layer, int n_head, int n_text_ctx) {
    std::string err;
    WLK_CHECK(make_tmap_bf16_2d(reinterpret_cast<CUtensorMap*>(tmap_out_host), self_kv,
                                (uint64_t)n_layer * 2 * n_head * n_text_ctx, DH, DH, BKV, DH, &err),
              "self-K/V tensor map: %s", err.c_str());
}

// causal self-attention of a decoder prefill on the tensor cores (bf16): every head, rows [0, n_rows) of each job at
// positions job.offset + row; the cache rows of this call were written by the QKV GEMM's scatter epilogue just before
void dec_self_attention_tcgen05(const void* q, int total_rows, const DecJob* jobs, int n_jobs, int max_rows, int layer,
                                int n_head, int d_model, int n_text_ctx, const void* kv_maps_dev, void* out, cudaStream_t st) {
    CUtensorMap tm;
    std::string err;
    WLK_CHECK(make_tmap_bf16_2d(&tm, q, (uint64_t)total_rows, (uint64_t)d_model, (uint64_t)d_model, BQ, DH, &err),
              "query tensor map: %s", err.c_str());
    static bool seen[64] = {};
    if (first_on_device(seen))
        CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel<MODE_SELF, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AttLayout<false>::SMEM));
    dim3 grid((max_rows + BQ - 1) / BQ, n_head, n_jobs);
    CUDA_CHECK(launch_pdl(attn_tc_kernel<MODE_SELF, false>, grid, dim3(ATT_THREADS), (size_t)AttLayout<false>::SMEM, st, tm, tm,
                          reinterpret_cast<const CUtensorMap*>(kv_maps_dev), jobs, layer, (const int32_t*)nullptr, n_head, d_model,
                          n_text_ctx, out));
}

}  // namespace wlk
