// wgmma GEMM for sm_90a:  C[M,N] = epilogue(A[M,K] * W[N,K]^T), bf16 operands, fp32 accumulate.
//
// Two kernels.  128 x 128 tiles (the encoder's GEMMs) run on the ping-pong kernel gemm_pp_kernel (below); the 64- and
// 32-wide tiles of short or narrow problems (the decoder's, with split-K) run on gemm_tc_kernel:
// persistent, warp-specialised, one CTA per SM:
//   warps 0..7  MMA + epilogue: two warpgroups, each owning 64 rows of the 128 x BN tile.  Per k-slab four
//                               wgmma.mma_async (M=64, N=BN, K=16) read both operands from shared memory and
//                               accumulate in registers, one slab in flight while the next is issued; then the
//                               fused bias / GELU / column scale / fp32 residual epilogue and bf16 or fp32
//                               stores (plain or scattered into the head-major KV layouts) from the fragment.
//   warp 8      TMA producer  : cp.async.bulk.tensor 2D loads of the A (128x64) and W (BNx64) k-slabs,
//                               128B-swizzled, into a STAGES-deep shared-memory ring (mbarrier full/empty);
//                               it keeps filling the ring with the next tile while the epilogue runs.
// Tiles are walked m-fastest so the CTAs of a wave share one W panel (L2-resident) while A streams.
#include <cudaTypedefs.h>

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <unordered_map>

#include "gemm_epi.cuh"

namespace wlk {

static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
    if (!g_encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        WLK_CHECK(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
        g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    }
    return g_encode;
}

// 2D bf16 (or fp32, or e4m3 bytes) tensor map over a row-major [rows, cols] matrix with row pitch ld (elements); box = [box_rows,
// box_cols], 128B-swizzled.  A descriptor is a pure function of (address, type, shape, pitch, box): the engine's
// workspaces and weights sit at fixed addresses, so the ~2 000 maps a tick needs are encoded once per calling thread
// and then served from a small thread-local table (no lock; unified addressing makes the pointer unique across devices).
namespace {
struct TmapKey {
    const void* ptr; uint64_t rows, cols, ld; uint32_t box_rows, box_cols; int dtype;
    bool operator==(const TmapKey& o) const {
        return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows &&
               box_cols == o.box_cols && dtype == o.dtype;
    }
};
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        uint64_t h = reinterpret_cast<uintptr_t>(k.ptr) * 0x9E3779B97F4A7C15ull;
        h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
        h ^= (k.cols * 1315423911ull + (h << 6) + (h >> 2));
        h ^= (k.ld * 2654435761ull + (h << 6) + (h >> 2));
        h ^= ((uint64_t)k.box_rows << 32 | k.box_cols) + (h << 6) + (h >> 2);
        h ^= (uint64_t)k.dtype + (h << 6) + (h >> 2);
        return (size_t)h;
    }
};

bool make_tmap_2d(CUtensorMap* tm, int dtype, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                  uint32_t box_rows, uint32_t box_cols, std::string* err) {
    static thread_local std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
    const TmapKey key{ptr, rows, cols, ld, box_rows, box_cols, dtype};
    auto it = cache.find(key);
    if (it != cache.end()) { *tm = it->second; return true; }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld * dtype_size(dtype)};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt = dtype == DT_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : dtype == DT_E4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    CUresult r = get_encode()(tm, dt, 2,
                              const_cast<void*>(ptr), gdim, gstride, box,
                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        if (err) *err = "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r);
        return false;
    }
    if (cache.size() >= 8192) cache.clear();      // decode prefills of every length each leave a few entries behind
    cache.emplace(key, *tm);
    return true;
}
}  // namespace

bool make_tmap_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols, std::string* err) {
    return make_tmap_2d(tm, DT_BF16, ptr, rows, cols, ld, box_rows, box_cols, err);
}

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int NUM_MMA_WARPS = 8;                        // two warpgroups, 64 rows of the tile each
constexpr int NUM_THREADS = 32 * NUM_MMA_WARPS + 32;    // + the TMA warp (last, so the warpgroups start at warp 0 and 4)


// X3 (WLK_PREC_BF16X3): every operand arrives as two bf16 planes, hi = bf16(x) and lo = bf16(x - hi); a k-slab stages
// four tiles (A_hi, A_lo, W_hi, W_lo) and every K=16 step issues three MMAs into the same fp32 accumulator:
// A_hi W_hi + A_lo W_hi + A_hi W_lo (the lo*lo term is below 2^-16 relative and dropped) -- ~16 mantissa bits per
// operand instead of 8, on the same tensor cores.
// EPI_BUFS: 16 KiB epilogue staging buffers behind the ring (the ping-pong kernel's TMA-store epilogue: two per
// consumer).
template <int BN, int STAGES, bool X3 = false, int EPI_BUFS = 0>
struct SmemLayout {
    static constexpr uint32_t PLANES = X3 ? 2 : 1;
    static constexpr uint32_t A_BYTES = BM * BK * 2;
    static constexpr uint32_t B_BYTES = BN * BK * 2;
    static constexpr uint32_t EPI_BYTES = 128 * 128;
    static constexpr uint32_t EPI_OFF = STAGES * PLANES * (A_BYTES + B_BYTES);     // 1024-aligned (128B swizzle)
    static constexpr uint32_t BAR_OFF = EPI_OFF + EPI_BUFS * EPI_BYTES;
    static constexpr uint32_t TOTAL = BAR_OFF + 2 * STAGES * 8 + 16;
    static constexpr uint32_t DYN = TOTAL + 1024;   // slack for manual 1024-byte alignment
};

template <int BN, int STAGES, bool X3>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmWlo, int M, int N, int K,
               int splits, float* __restrict__ sk_scratch, int* __restrict__ sk_counters, Epilogue epi) {
    using L = SmemLayout<BN, STAGES, X3>;
    constexpr uint32_t STAGE_TX = L::PLANES * (L::A_BYTES + L::B_BYTES);
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));
    const uint32_t sA = smem_base;
    const uint32_t sB = smem_base + STAGES * L::A_BYTES;
    const uint32_t sAlo = sB + STAGES * L::B_BYTES;                // X3 only
    const uint32_t sBlo = sAlo + STAGES * L::A_BYTES;              // X3 only
    const uint32_t bar_full = smem_base + L::BAR_OFF;              // [STAGES]
    const uint32_t bar_empty = bar_full + STAGES * 8;              // [STAGES]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_m = (M + BM - 1) / BM, num_n = (N + BN - 1) / BN;
    const int num_mn = num_m * num_n;
    const int num_tiles = num_mn * splits;            // split-K: a work item is (k-range, n block, m block)
    const int num_k_total = (K + BK - 1) / BK;
    const int kb_per_split = (num_k_total + splits - 1) / splits;
    const int band = max(1, (int)gridDim.x / 2);

    ptx::griddep_launch();
    if (warp == NUM_MMA_WARPS && lane == 0) {
        ptx::prefetch_tensormap(&tmA);
        ptx::prefetch_tensormap(&tmW);
        if (X3) { ptx::prefetch_tensormap(&tmAlo); ptx::prefetch_tensormap(&tmWlo); }
        for (int i = 0; i < STAGES; ++i) {
            ptx::mbar_init(bar_full + 8 * i, 1);
            ptx::mbar_init(bar_empty + 8 * i, NUM_MMA_WARPS);      // lane 0 of every MMA warp releases a slot
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == NUM_MMA_WARPS) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            // The weight panels never depend on the previous kernel: the first ring-full of them is requested
            // before the grid-dependency wait, so under programmatic dependent launch the weight stream of this
            // GEMM overlaps the tail of whatever produced its activations.  `early` counts those k-blocks.
            int early = 0;
            if ((int)blockIdx.x < num_tiles) {
                const int sp = blockIdx.x / num_mn, mn = blockIdx.x - sp * num_mn;
                int m_blk, n_blk;
                tile_coords(mn, num_m, num_n, band, &m_blk, &n_blk);
                const int kb0 = sp * kb_per_split;
                early = min(STAGES, min(num_k_total, (sp + 1) * kb_per_split) - kb0);
                for (int i = 0; i < early; ++i) {
                    ptx::mbar_arrive_expect_tx(bar_full + 8 * i, STAGE_TX);
                    ptx::tma_load_2d(sB + i * L::B_BYTES, &tmW, bar_full + 8 * i, (kb0 + i) * BK, n_blk * BN);
                    if (X3) ptx::tma_load_2d(sBlo + i * L::B_BYTES, &tmWlo, bar_full + 8 * i, (kb0 + i) * BK, n_blk * BN);
                }
            }
            ptx::griddep_wait();
            uint32_t stage = 0, phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int sp = tile / num_mn, mn = tile - sp * num_mn;
                int m_blk, n_blk;
                tile_coords(mn, num_m, num_n, band, &m_blk, &n_blk);
                const int kb_end = min(num_k_total, (sp + 1) * kb_per_split);
                for (int kb = sp * kb_per_split; kb < kb_end; ++kb) {
                    if (early > 0) {
                        --early;                       // slot is fresh and its W panel is already in flight
                    } else {
                        ptx::mbar_wait_mma(bar_empty + 8 * stage, phase ^ 1);
                        ptx::mbar_arrive_expect_tx(bar_full + 8 * stage, STAGE_TX);
                        ptx::tma_load_2d(sB + stage * L::B_BYTES, &tmW, bar_full + 8 * stage, kb * BK, n_blk * BN);
                        if (X3) ptx::tma_load_2d(sBlo + stage * L::B_BYTES, &tmWlo, bar_full + 8 * stage, kb * BK, n_blk * BN);
                    }
                    ptx::tma_load_2d(sA + stage * L::A_BYTES, &tmA, bar_full + 8 * stage, kb * BK, m_blk * BM);
                    if (X3) ptx::tma_load_2d(sAlo + stage * L::A_BYTES, &tmAlo, bar_full + 8 * stage, kb * BK, m_blk * BM);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== MMA + epilogue (warps 0..7) =====================
        // The producer runs ahead through the ring, so the next tile's first k-slabs land while this one's epilogue runs.
        const int wg = warp >> 2, wq = warp & 3;
        constexpr uint32_t WG_A_OFF = 64 * BK * 2;          // the warpgroup's 64 rows of the 128-row A tile
        volatile int* sk_flag = reinterpret_cast<volatile int*>(smem_gen + L::BAR_OFF + 2 * STAGES * 8);
        uint32_t stage = 0, phase = 0;
        ptx::griddep_wait();                          // residual, split-K scratch and C belong to the stream's past
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int sp = tile / num_mn, mn = tile - sp * num_mn;
            int m_blk, n_blk;
            tile_coords(mn, num_m, num_n, band, &m_blk, &n_blk);
            const int row0 = m_blk * BM + wg * 64 + wq * 16 + (lane >> 2);
            const EpiRow rows[2] = {epi_row(epi, row0, M), epi_row(epi, row0 + 8, M)};
            epilogue_prefetch_residual(rows[0], n_blk * BN, BN, N);
            epilogue_prefetch_residual(rows[1], n_blk * BN, BN, N);
            const int kb_begin = sp * kb_per_split, kb_end = min(num_k_total, (sp + 1) * kb_per_split);
            float acc[BN / 2];
            int prev = -1;                            // slot whose MMAs are still in flight
            for (int kb = kb_begin; kb < kb_end; ++kb) {
                ptx::mbar_wait_mma(bar_full + 8 * stage, phase);
                const uint64_t da = ptx::wgmma_desc_sw128(sA + stage * L::A_BYTES + wg * WG_A_OFF);
                const uint64_t db = ptx::wgmma_desc_sw128(sB + stage * L::B_BYTES);
                const uint64_t dal = ptx::wgmma_desc_sw128(sAlo + stage * L::A_BYTES + wg * WG_A_OFF);
                const uint64_t dbl = ptx::wgmma_desc_sw128(sBlo + stage * L::B_BYTES);
                ptx::wgmma_fence_regs(acc);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    // advancing K by 16 bf16 = 32 bytes = +2 in the (addr >> 4) field
                    ptx::WgmmaSS<BN>::mma(acc, da + 2 * k, db + 2 * k, (kb > kb_begin || k > 0) ? 1u : 0u);
                    if (X3) {
                        ptx::WgmmaSS<BN>::mma(acc, dal + 2 * k, db + 2 * k, 1u);
                        ptx::WgmmaSS<BN>::mma(acc, da + 2 * k, dbl + 2 * k, 1u);
                    }
                }
                ptx::wgmma_commit();
                ptx::wgmma_wait<1>();                 // the previous slab's MMAs have retired: its slot is free
                if (prev >= 0 && lane == 0) ptx::mbar_arrive(bar_empty + 8 * prev);
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_regs(acc);
            if (prev >= 0 && lane == 0) ptx::mbar_arrive(bar_empty + 8 * prev);
            if (splits > 1) {
                // Split-K with a serial fix-up: every CTA of a tile parks its raw partial sums in global scratch;
                // the one that arrives last (atomic ticket) adds the others to its own accumulators and runs the
                // normal fused epilogue, so any output type / scatter mode works.
                const int64_t split_stride = (int64_t)num_mn * BM * BN;
                float* tile0 = sk_scratch + (int64_t)mn * BM * BN + (int64_t)wg * 64 * BN;
                partials_store<BN>(tile0 + sp * split_stride, acc, wq, lane);
                __threadfence();
                asm volatile("bar.sync 1, %0;" ::"n"(32 * NUM_MMA_WARPS) : "memory");
                if (warp == 0 && lane == 0) {
                    const int old = atomicAdd(sk_counters + mn, 1);
                    const int last = (old == splits - 1);
                    if (last) sk_counters[mn] = 0;                    // every split has arrived: re-arm for the next launch
                    *sk_flag = last;
                }
                asm volatile("bar.sync 1, %0;" ::"n"(32 * NUM_MMA_WARPS) : "memory");
                const int last = *sk_flag;
                asm volatile("bar.sync 1, %0;" ::"n"(32 * NUM_MMA_WARPS) : "memory");   // flag may be rewritten next tile
                if (!last) continue;
                __threadfence();
                for (int s2 = 0; s2 < splits; ++s2)
                    if (s2 != sp) partials_add<BN>(tile0 + s2 * split_stride, acc, wq, lane);
            }
            epilogue_fragment_tile<BN>(epi, rows, acc, n_blk * BN, N, lane);
        }
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// Ping-pong kernel for 128 x 128 tiles (the encoder GEMMs): three warpgroups, persistent, one CTA per SM.
//   WG0      TMA producer: one thread fills the ring with the k-slabs of the CTA's tiles in walk order; the warpgroup
//            gives registers back (setmaxnreg.dec).
//   WG1, WG2 consumers (setmaxnreg.inc): each owns a whole 128 x 128 tile -- two m64n128k16 wgmmas per K16 step,
//            128 fp32 accumulators per thread -- and they take alternate tiles of the walk.  A named-barrier handoff
//            orders their mainloops: a consumer issues its tile's MMAs only after the other has issued all of its own,
//            then runs its epilogue while the other's MMAs keep the tensor pipe busy.
// The producer fills the ring in the interleaved tile order, so a consumer's j-th tile of the walk starts at k-slab
// j * num_k of the ring's sequence (every tile has num_k slabs: no split-K here); it skips the other consumer's slabs by
// recomputing stage and phase from that count.  Each output element is accumulated in the same K order as in
// gemm_tc_kernel.
//
// Clusters (CM x CN CTAs, CM * CN > 1): the cluster owns a CM x CN block of tiles (a cluster-tile) and walks the
// cluster-tiles as a lone CTA walks tiles; CTA rank r takes tile (rm, rn) = (r % CM, r / CM) of each.  The CM CTAs of an
// n column need the same W slab and the CN CTAs of an m row the same A slab, so each loads 1/CM of the W slab and
// 1/CN of the A slab and multicasts its share to the CTAs that need it: a slab is read from L2 once per cluster instead
// of once per CTA.  Every CTA's full barrier still expects the whole stage.  A stage is refilled only when the consumers
// of every CTA of the cluster have released it (each consumer warp arrives on the empty barrier of every CTA), so the
// CTAs of a cluster run the same slab sequence in lockstep.  A tile past M or N (odd num_m) is loaded (TMA zero-fills
// it), computed and released like any other; its epilogue stores nothing.  <STAGES, X3, 1, 1> is the lone-CTA kernel.
//
// TMA_C: plain row-major outputs without a residual that a tensor map can address (the encoder's conv1, QKV and FC1)
// leave through epilogue_tma_tile128: each consumer stages its tile in two 16 KiB shared-memory buffers and stores it
// by TMA (tmC).  The scatter modes and the fp32 residual outputs keep the register-path epilogue (epilogue_tile128) and
// the deeper ring (see tma_epilogue_fits).
constexpr int PP_THREADS = 3 * 128;
constexpr int PP_PRODUCER_REGS = 40, PP_CONSUMER_REGS = 232;     // 128 * 40 + 256 * 232 <= 64K registers
constexpr int PP_BAR_ORDER = 1;                                  // named barriers 1, 2: "consumer c may issue its MMAs"
constexpr int PP_BAR_EPI = 3;                                    // named barriers 3, 4: consumer c's staged epilogue
// L2 budget for the A rows of one m-band (tile_coords): with two tiles in flight per CTA the band is swept across
// ~2 x grid tiles at a time, and its A rows should be served from L2 for the whole sweep over n
constexpr int64_t PP_BAND_BYTES = 20ll << 20;

template <int STAGES, bool X3, int CM, int CN, bool TMA_C, bool FP8>
__global__ void __launch_bounds__(PP_THREADS, 1)
gemm_pp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmWlo,
               const __grid_constant__ CUtensorMap tmC, int M, int N, int K,
               Epilogue epi) {
    constexpr int BN = 128;
    constexpr int KE = FP8 ? 2 * BK : BK;                          // K elements per 128-byte slab row
    constexpr int CS = CM * CN;                                    // CTAs per cluster
    constexpr int W_ROWS = BN / CM, A_ROWS = BM / CN;              // this CTA's share of a W / A slab (the tensor maps' box)
    using L = SmemLayout<BN, STAGES, X3, TMA_C ? 4 : 0>;
    constexpr uint32_t STAGE_TX = L::PLANES * (L::A_BYTES + L::B_BYTES);
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem_base;
    const uint32_t sB = smem_base + STAGES * L::A_BYTES;
    const uint32_t sAlo = sB + STAGES * L::B_BYTES;                // X3 only
    const uint32_t sBlo = sAlo + STAGES * L::A_BYTES;              // X3 only
    const uint32_t bar_full = smem_base + L::BAR_OFF;              // [STAGES]
    const uint32_t bar_empty = bar_full + STAGES * 8;              // [STAGES]

    const int wg = threadIdx.x >> 7;
    const int rank = CS > 1 ? (int)ptx::cluster_ctarank() : 0;
    const int rm = rank % CM, rn = rank / CM;
    const int cluster = CS > 1 ? (int)ptx::cluster_id_x() : (int)blockIdx.x;
    const int clusters = CS > 1 ? (int)ptx::num_clusters_x() : (int)gridDim.x;
    const int num_m = (M + BM - 1) / BM, num_n = (N + BN - 1) / BN;
    const int cnum_m = (num_m + CM - 1) / CM, cnum_n = (num_n + CN - 1) / CN;
    const int num_ct = cnum_m * cnum_n;                            // cluster-tiles
    const int num_k = (K + KE - 1) / KE;
    auto coords = [&](int ct, int* m_blk, int* n_blk) {
        // (recomputed per tile in 32-bit arithmetic rather than held in a register across the consumers' tile loop)
        const int band_fit = (int)((uint32_t)PP_BAND_BYTES / ((uint32_t)CM * BM * (FP8 ? 1 : 2) * L::PLANES * (uint32_t)K));
        const int band = max(1, min(2 * clusters, band_fit));
        tile_coords(ct, cnum_m, cnum_n, band, m_blk, n_blk);
        *m_blk = *m_blk * CM + rm;
        *n_blk = *n_blk * CN + rn;
    };

    ptx::griddep_launch();
    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tmA);
        ptx::prefetch_tensormap(&tmW);
        if (X3) { ptx::prefetch_tensormap(&tmAlo); ptx::prefetch_tensormap(&tmWlo); }
        for (int i = 0; i < STAGES; ++i) {
            ptx::mbar_init(bar_full + 8 * i, 1);
            ptx::mbar_init(bar_empty + 8 * i, 4 * CS);             // lane 0 of each warp of the consuming warpgroups
        }
        if (TMA_C) ptx::prefetch_tensormap(&tmC);
        ptx::fence_barrier_init();
    }
    // the peers' barriers must be initialised before the first multicast lands on them
    if (CS > 1) ptx::cluster_sync();
    else __syncthreads();

    if (wg == 0) {
        // ===================== TMA producer =====================
        ptx::setmaxnreg_dec<PP_PRODUCER_REGS>();
        if (threadIdx.x == 0) {
            uint16_t w_mask = 0, a_mask = 0;                       // the CTAs of this one's n column / m row
            for (int i = 0; i < CM; ++i) w_mask |= 1u << (rn * CM + i);
            for (int i = 0; i < CN; ++i) a_mask |= 1u << (i * CM + rm);
            // this CTA's share of a slab: rows [rm * W_ROWS, +W_ROWS) of the W tile, [rn * A_ROWS, +A_ROWS) of the A tile
            auto load = [&](uint32_t dst, const CUtensorMap* tm, uint32_t bar, int kb, int row, uint16_t mask, bool shared) {
                if (shared) ptx::tma_load_2d_multicast(dst, tm, bar, kb * KE, row, mask);
                else ptx::tma_load_2d(dst, tm, bar, kb * KE, row);
            };
            auto load_w = [&](uint32_t stage, int kb, int n_blk) {
                const uint32_t off = stage * L::B_BYTES + rm * W_ROWS * BK * 2, bar = bar_full + 8 * stage;
                load(sB + off, &tmW, bar, kb, n_blk * BN + rm * W_ROWS, w_mask, CM > 1);
                if (X3) load(sBlo + off, &tmWlo, bar, kb, n_blk * BN + rm * W_ROWS, w_mask, CM > 1);
            };
            auto load_a = [&](uint32_t stage, int kb, int m_blk) {
                const uint32_t off = stage * L::A_BYTES + rn * A_ROWS * BK * 2, bar = bar_full + 8 * stage;
                load(sA + off, &tmA, bar, kb, m_blk * BM + rn * A_ROWS, a_mask, CN > 1);
                if (X3) load(sAlo + off, &tmAlo, bar, kb, m_blk * BM + rn * A_ROWS, a_mask, CN > 1);
            };
            // the first ring-full of weight panels does not depend on the previous kernel: requested before the
            // grid-dependency wait (see gemm_tc_kernel)
            int early = 0;
            if (cluster < num_ct) {
                int m_blk, n_blk;
                coords(cluster, &m_blk, &n_blk);
                early = min(STAGES, num_k);
                for (int i = 0; i < early; ++i) {
                    ptx::mbar_arrive_expect_tx(bar_full + 8 * i, STAGE_TX);
                    load_w(i, i, n_blk);
                }
            }
            ptx::griddep_wait();
            uint32_t stage = 0, phase = 0;
            for (int ct = cluster; ct < num_ct; ct += clusters) {
                int m_blk, n_blk;
                coords(ct, &m_blk, &n_blk);
                for (int kb = 0; kb < num_k; ++kb) {
                    if (early > 0) {
                        --early;
                    } else {
                        ptx::mbar_wait_mma(bar_empty + 8 * stage, phase ^ 1);
                        ptx::mbar_arrive_expect_tx(bar_full + 8 * stage, STAGE_TX);
                        load_w(stage, kb, n_blk);
                    }
                    load_a(stage, kb, m_blk);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumers: MMA + epilogue =====================
        ptx::setmaxnreg_inc<PP_CONSUMER_REGS>();
        const int c = wg - 1;
        const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
        constexpr uint32_t HALF_A = 64 * BK * 2;                   // rows 64..127 of the A tile (+HALF_A >> 4 in a descriptor)
        // a stage is free again once this warp is done with it: lane i tells cluster rank i, whose producer may multicast into it
        auto release = [&](uint32_t stage) {
            if (CS > 1) { if (lane < CS) ptx::mbar_arrive_cluster(bar_empty + 8 * stage, lane); }
            else if (lane == 0) ptx::mbar_arrive(bar_empty + 8 * stage);
        };
        ptx::griddep_wait();                                       // residual and C belong to the stream's past
        for (int ct = cluster + c * clusters; ct < num_ct; ct += 2 * clusters) {
            const int j = (ct - cluster) / clusters;               // position of the tile in the CTA's walk
            int m_blk, n_blk;
            coords(ct, &m_blk, &n_blk);
            const int row0 = m_blk * BM + wq * 16 + (lane >> 2);
            const uint32_t slab0 = (uint32_t)j * num_k;
            uint32_t stage = slab0 % STAGES, phase = (slab0 / STAGES) & 1;
            float acc[2][64];
            int prev = -1;                                         // slot whose MMAs are still in flight
            if (j > 0) ptx::named_bar_sync<256>(PP_BAR_ORDER + c);  // the other consumer has issued its tile
            for (int kb = 0; kb < num_k; ++kb) {
                ptx::mbar_wait_mma(bar_full + 8 * stage, phase);
                const uint64_t da = ptx::wgmma_desc_sw128(sA + stage * L::A_BYTES);
                const uint64_t db = ptx::wgmma_desc_sw128(sB + stage * L::B_BYTES);
                const uint64_t dal = ptx::wgmma_desc_sw128(sAlo + stage * L::A_BYTES);
                const uint64_t dbl = ptx::wgmma_desc_sw128(sBlo + stage * L::B_BYTES);
                ptx::wgmma_fence_regs(acc[0]);
                ptx::wgmma_fence_regs(acc[1]);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint32_t acc_in = (kb > 0 || k > 0) ? 1u : 0u;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint64_t ah = h * (HALF_A >> 4) + 2 * k;
                        if (FP8) ptx::wgmma_e4m3_n128(acc[h], da + ah, db + 2 * k, acc_in);   // K = 32 e4m3: 32 bytes too
                        else ptx::WgmmaSS<BN>::mma(acc[h], da + ah, db + 2 * k, acc_in);
                        if (X3) {
                            ptx::WgmmaSS<BN>::mma(acc[h], dal + ah, db + 2 * k, 1u);
                            ptx::WgmmaSS<BN>::mma(acc[h], da + ah, dbl + 2 * k, 1u);
                        }
                    }
                }
                ptx::wgmma_commit();
                ptx::wgmma_wait<1>();                              // the previous slab's MMAs have retired: its slot is free
                if (prev >= 0) release(prev);
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            if (ct + clusters < num_ct) ptx::named_bar_arrive<256>(PP_BAR_ORDER + (c ^ 1));   // the next tile's turn
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_regs(acc[0]);
            ptx::wgmma_fence_regs(acc[1]);
            release(prev);
            if (!TMA_C) {
                epilogue_tile128<FP8>(epi, row0, M, acc, n_blk * BN, N, lane);
            } else if (m_blk * BM < M && n_blk * BN < N) {         // (not a cluster-padding tile)
                epilogue_math_tile128<FP8>(epi, acc, n_blk * BN, N, lane, row0, M);
                const uint32_t buf = smem_base + L::EPI_OFF + c * 2 * L::EPI_BYTES;   // the consumer's two buffers
                if (epi.c_type == DT_F32) epilogue_tma_tile128<4>(acc, &tmC, m_blk * BM, n_blk * BN, buf, PP_BAR_EPI + c, wq, lane);
                else if (FP8 && epi.c_type == DT_E4M3) {
                    epilogue_out_scale_tile128(epi, row0, M, acc);
                    epilogue_tma_tile128<1>(acc, &tmC, m_blk * BM, n_blk * BN, buf, PP_BAR_EPI + c, wq, lane);
                } else epilogue_tma_tile128<2>(acc, &tmC, m_blk * BM, n_blk * BN, buf, PP_BAR_EPI + c, wq, lane);
            }
        }
        // the tile stores have written global memory before the CTA exits (the next kernel's griddepcontrol.wait and
        // the cluster's exit barrier rely on it)
        if (TMA_C && threadIdx.x % 128 == 0) ptx::bulk_wait_group<0>();
    }
    // no CTA may exit while a peer can still arrive on its barriers
    if (CS > 1) ptx::cluster_sync();
}

// fp32 -> (hi, lo) bf16 planes: hi = bf16(x), lo = bf16(x - hi)
__global__ void split_f32_kernel(const float* __restrict__ src, bf16* __restrict__ hi, bf16* __restrict__ lo, int64_t n) {
    ptx::griddep_launch();
    ptx::griddep_wait();
    const int64_t n4 = n >> 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 v = reinterpret_cast<const float4*>(src)[i];
        const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
        const __nv_bfloat162 l0 = __floats2bfloat162_rn(v.x - __low2float(h0), v.y - __high2float(h0));
        const __nv_bfloat162 l1 = __floats2bfloat162_rn(v.z - __low2float(h1), v.w - __high2float(h1));
        uint2 uh, ul;
        uh.x = *reinterpret_cast<const uint32_t*>(&h0); uh.y = *reinterpret_cast<const uint32_t*>(&h1);
        ul.x = *reinterpret_cast<const uint32_t*>(&l0); ul.y = *reinterpret_cast<const uint32_t*>(&l1);
        reinterpret_cast<uint2*>(hi)[i] = uh;
        reinterpret_cast<uint2*>(lo)[i] = ul;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const int64_t i = (n4 << 2) + threadIdx.x;
        const bf16 h = __float2bfloat16_rn(src[i]);
        hi[i] = h;
        lo[i] = __float2bfloat16_rn(src[i] - __bfloat162float(h));
    }
}

template <int BN, int STAGES, bool X3>
void launch_impl(const GemmArgs& g, const void* A_hi, const void* A_lo, cudaStream_t st, int num_sms, int splits) {
    using L = SmemLayout<BN, STAGES, X3>;
    static_assert(L::DYN <= 227 * 1024, "shared memory budget");
    if (splits > 1) {
        const int tiles_mn = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN);
        // the partial-tile scratch and the ticket counters belong to the calling engine (GemmArgs): two engines on one
        // device never share them
        if (!g.sk_scratch || !g.sk_counters || (size_t)splits * tiles_mn * BM * BN > g.sk_scratch_floats ||
            tiles_mn > g.sk_max_tiles)
            splits = 1;
    }
    CUtensorMap tmA, tmW, tmAlo, tmWlo;
    std::string err;
    WLK_CHECK(make_tmap_bf16_2d(&tmA, A_hi, g.M, g.K, g.lda, BM, BK, &err), "A tensor map: %s", err.c_str());
    WLK_CHECK(make_tmap_bf16_2d(&tmW, g.W, g.N, g.K, g.ldw, BN, BK, &err), "W tensor map: %s", err.c_str());
    if (X3) {
        WLK_CHECK(make_tmap_bf16_2d(&tmAlo, A_lo, g.M, g.K, g.lda, BM, BK, &err), "A_lo tensor map: %s", err.c_str());
        WLK_CHECK(make_tmap_bf16_2d(&tmWlo, g.W_lo, g.N, g.K, g.ldw, BN, BK, &err), "W_lo tensor map: %s", err.c_str());
    } else { tmAlo = tmA; tmWlo = tmW; }
    static bool seen[64] = {};
    if (first_on_device(seen))
        CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<BN, STAGES, X3>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)L::DYN));
    const int num_tiles = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN) * splits;
    const int grid = num_tiles < num_sms ? num_tiles : num_sms;
    CUDA_CHECK(launch_pdl(gemm_tc_kernel<BN, STAGES, X3>, dim3(grid), dim3(NUM_THREADS), L::DYN, st, tmA, tmW, tmAlo, tmWlo,
                          g.M, g.N, g.K, splits, g.sk_scratch, g.sk_counters, g.epi));
}

// STAGES / STAGES3: ring depth of the plain and of the X3 instantiation (four tiles per slab: half the depth)
template <int BN, int STAGES, int STAGES3>
void launch(const GemmArgs& g, const void* A_hi, const void* A_lo, cudaStream_t st, int num_sms, int splits = 1) {
    if (g.w_type == DT_BF16X2) launch_impl<BN, STAGES3, true>(g, A_hi, A_lo, st, num_sms, splits);
    else launch_impl<BN, STAGES, false>(g, A_hi, A_lo, st, num_sms, splits);
}

template <int STAGES, bool X3, int CM, int CN, bool TMA_C, bool FP8 = false>
void launch_pp_impl(const GemmArgs& g, const void* A_hi, const void* A_lo, cudaStream_t st, int num_sms) {
    using L = SmemLayout<128, STAGES, X3, TMA_C ? 4 : 0>;
    static_assert(L::DYN <= 227 * 1024, "shared memory budget");
    constexpr int CS = CM * CN;
    auto kernel = gemm_pp_kernel<STAGES, X3, CM, CN, TMA_C, FP8>;
    // each CTA loads 1/CN of an A slab and 1/CM of a W slab (the kernel's multicast shares); a slab row is 128 bytes
    constexpr int OP = FP8 ? DT_E4M3 : DT_BF16;
    constexpr uint32_t KE = FP8 ? 2 * BK : BK;
    CUtensorMap tmA, tmW, tmAlo, tmWlo;
    std::string err;
    WLK_CHECK(make_tmap_2d(&tmA, OP, A_hi, g.M, g.K, g.lda, BM / CN, KE, &err), "A tensor map: %s", err.c_str());
    WLK_CHECK(make_tmap_2d(&tmW, OP, g.W, g.N, g.K, g.ldw, 128 / CM, KE, &err), "W tensor map: %s", err.c_str());
    if (X3) {
        WLK_CHECK(make_tmap_bf16_2d(&tmAlo, A_lo, g.M, g.K, g.lda, BM / CN, BK, &err), "A_lo tensor map: %s", err.c_str());
        WLK_CHECK(make_tmap_bf16_2d(&tmWlo, g.W_lo, g.N, g.K, g.ldw, 128 / CM, BK, &err), "W_lo tensor map: %s", err.c_str());
    } else { tmAlo = tmA; tmWlo = tmW; }
    // the staged epilogue's sub-tiles: 128 rows x 128 bytes of C
    CUtensorMap tmC = tmA;
    if (TMA_C)
        WLK_CHECK(make_tmap_2d(&tmC, g.epi.c_type, g.epi.C, g.M, g.N, g.epi.ldc, BM, 128 / dtype_size(g.epi.c_type), &err),
                  "C tensor map: %s", err.c_str());
    // clusters of this shape the device holds at once (it depends on how the SMs split into GPCs): queried once per device
    static std::atomic<int> max_clusters[64];
    const int dev = current_device();
    int mc = max_clusters[dev].load(std::memory_order_relaxed);
    if (mc == 0) {
        CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L::DYN));
        mc = num_sms;
        if (CS > 1) {
            cudaLaunchConfig_t cfg = {};
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = CS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
            cfg.gridDim = dim3(CS);
            cfg.blockDim = dim3(PP_THREADS);
            cfg.dynamicSmemBytes = L::DYN;
            cfg.attrs = attr;
            cfg.numAttrs = 1;
            CUDA_CHECK(cudaOccupancyMaxActiveClusters(&mc, kernel, &cfg));
            WLK_CHECK(mc > 0, "no %dx%d cluster of the 128-wide GEMM fits on the device", CM, CN);
        }
        max_clusters[dev].store(mc, std::memory_order_relaxed);
    }
    const int num_ct = ((g.M + BM * CM - 1) / (BM * CM)) * ((g.N + 128 * CN - 1) / (128 * CN));
    const int clusters = std::max(1, std::min({mc, num_sms / CS, num_ct}));
    CUDA_CHECK(launch_pdl_cluster(kernel, dim3(clusters * CS), dim3(PP_THREADS), L::DYN, st, CS, tmA, tmW, tmAlo, tmWlo,
                                  tmC, g.M, g.N, g.K, g.epi));
}

// Whether the ping-pong kernel's staged epilogue writes C: a plain row-major output at a 16-byte aligned base and pitch
// (what a tensor map can address), without a residual.  The fp32 residual outputs (attention-out and FC2, x += A W^T in
// place) stay on the register path and its 6-stage ring: with the residual staged through the same buffers by TMA they
// measured 3-9 % slower (DESIGN.md section 3).
bool tma_epilogue_fits(const Epilogue& e) {
    return e.mode == EPI_PLAIN && e.residual == nullptr && reinterpret_cast<uintptr_t>(e.C) % 16 == 0 &&
           (e.ldc * (int64_t)dtype_size(e.c_type)) % 16 == 0;
}

// 128 x 128 tiles on the ping-pong kernel, in clusters of CM x CN CTAs.  Ring depth 3 for X3 (four tiles per slab);
// otherwise 6, or 5 beside the staged epilogue's 64 KiB of buffers; e4m3 operands (FP8) use the same ring.
template <int CM, int CN>
void launch_pp(const GemmArgs& g, const void* A_hi, const void* A_lo, cudaStream_t st, int num_sms) {
    if (g.w_type == DT_BF16X2) launch_pp_impl<3, true, 1, 1, false>(g, A_hi, A_lo, st, num_sms);
    else if (g.w_type == DT_E4M3 && tma_epilogue_fits(g.epi)) launch_pp_impl<5, false, CM, CN, true, true>(g, A_hi, A_lo, st, num_sms);
    else if (g.w_type == DT_E4M3) launch_pp_impl<6, false, CM, CN, false, true>(g, A_hi, A_lo, st, num_sms);
    else if (tma_epilogue_fits(g.epi)) launch_pp_impl<5, false, CM, CN, true>(g, A_hi, A_lo, st, num_sms);
    else launch_pp_impl<6, false, CM, CN, false>(g, A_hi, A_lo, st, num_sms);
}

}  // namespace

void split_f32_planes_async(const float* src, bf16* hi, bf16* lo, int64_t n, cudaStream_t st) {
    int grid = (int)std::min<int64_t>((n / 4 + 255) / 256, 132 * 8);
    if (grid < 1) grid = 1;
    CUDA_CHECK(launch_pdl(split_f32_kernel, dim3(grid), dim3(256), 0, st, src, hi, lo, n));
}

bool gemm_tcgen05_supported(const GemmArgs& g, std::string* why) {
    auto fail = [&](const char* m) { if (why) *why = m; return false; };
    const bool x3 = g.w_type == DT_BF16X2;
    if (g.a_type == DT_E4M3 || g.w_type == DT_E4M3) {
        // e4m3: 128-wide ping-pong kernel only, K-major operands with a 16-byte pitch, the scales present
        if (g.a_type != DT_E4M3 || g.w_type != DT_E4M3) return fail("e4m3: both operands must be e4m3");
        if (reinterpret_cast<uintptr_t>(g.A) % 16 || reinterpret_cast<uintptr_t>(g.W) % 16)
            return fail("operands must be 16-byte aligned");
        if (g.lda % 16 || g.ldw % 16) return fail("e4m3: row pitch must be a multiple of 16 elements (16 bytes)");
        if (g.K % 16) return fail("e4m3: K must be a multiple of 16");
        if (!g.epi.a_scale || !g.epi.w_scale) return fail("e4m3: operand scales missing");
        if (g.epi.c_type == DT_E4M3 && (!g.epi.c_scale || !tma_epilogue_fits(g.epi)))
            return fail("e4m3 output: plain rows at a 16-byte aligned base and pitch, no residual, with a row scale");
        if (g.M <= 0 || g.N <= 0 || g.K <= 0) return fail("empty problem");
        return true;
    }
    if (g.epi.c_type == DT_E4M3) return fail("an e4m3 output needs e4m3 operands");
    if (x3) {
        if (g.a_type != DT_F32) return fail("bf16x3: the activation operand must be fp32 (it is split on the fly)");
        if (!g.W_lo) return fail("bf16x3: missing lo plane of the weights");
        const size_t need = (size_t)(g.M - 1) * g.lda + g.K;
        if (!g.a_split || need > g.a_split_elems) return fail("bf16x3: split scratch missing or too small");
        if (reinterpret_cast<uintptr_t>(g.A) % 16) return fail("operands must be 16-byte aligned");
    } else {
        if (g.a_type != DT_BF16 || g.w_type != DT_BF16) return fail("operands must be bf16");
        if (reinterpret_cast<uintptr_t>(g.A) % 16) return fail("operands must be 16-byte aligned");
    }
    if (g.lda % 8 || g.ldw % 8) return fail("row pitch must be a multiple of 8 elements (16 bytes)");
    if (reinterpret_cast<uintptr_t>(g.W) % 16) return fail("operands must be 16-byte aligned");
    if (g.K % 8) return fail("K must be a multiple of 8");
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) return fail("empty problem");
    return true;
}

void gemm_tcgen05(const GemmArgs& g, cudaStream_t st, int num_sms, int variant) {
    std::string why;
    WLK_CHECK(gemm_tcgen05_supported(g, &why), "gemm_tcgen05: %s", why.c_str());
    static const int forced = [] { const char* v = getenv("WLK_GEMM_VARIANT"); return v ? atoi(v) : 0; }();
    if (variant == 0) variant = forced;
    const void *A_hi = g.A, *A_lo = nullptr;
    if (g.w_type == DT_BF16X2) {
        // split the fp32 activation operand (the whole underlying range: conv views have overlapping rows, lda < K)
        const int64_t n = (int64_t)(g.M - 1) * g.lda + g.K;
        bf16* hi = reinterpret_cast<bf16*>(g.a_split);
        bf16* lo = hi + g.a_split_elems;
        split_f32_planes_async(reinterpret_cast<const float*>(g.A), hi, lo, n, st);
        A_hi = hi; A_lo = lo;
    }
    // forced tile width / split-K (op-level tests, WLK_GEMM_VARIANT): 1 = <64,8>, 2 = 128-wide ping-pong on lone CTAs,
    // 4 = <32,10>, 5/6 = <64,8> split-K 2/4, 7/8 = <32,10> split-K 2/4, 9/10/11 = 128-wide in 2x1 / 1x2 / 2x2 clusters
    if (g.w_type == DT_E4M3) {
        // e4m3 runs on the 128-wide kernel only, unsplit (deterministic, batch-invariant): 2x2 clusters from K = 1024 when
        // the tiles cover half the SMs, lone CTAs otherwise (the conv-free short K, the incremental encoder's blocks)
        WLK_CHECK(variant == 0 || variant == 2 || (variant >= 9 && variant <= 11),
                  "gemm_tcgen05: variant %d has no e4m3 kernel (e4m3 runs on the 128-wide ping-pong kernel only)", variant);
        const int tiles = ((g.M + BM - 1) / BM) * ((g.N + 127) / 128);
        if (variant == 9) launch_pp<2, 1>(g, A_hi, A_lo, st, num_sms);
        else if (variant == 10) launch_pp<1, 2>(g, A_hi, A_lo, st, num_sms);
        else if (variant == 11 || (variant == 0 && g.K >= 1024 && tiles >= num_sms / 2)) launch_pp<2, 2>(g, A_hi, A_lo, st, num_sms);
        else launch_pp<1, 1>(g, A_hi, A_lo, st, num_sms);
        return;
    }
    if (variant == 2) { launch_pp<1, 1>(g, A_hi, A_lo, st, num_sms); return; }
    if (variant == 9) { launch_pp<2, 1>(g, A_hi, A_lo, st, num_sms); return; }
    if (variant == 10) { launch_pp<1, 2>(g, A_hi, A_lo, st, num_sms); return; }
    if (variant == 11) { launch_pp<2, 2>(g, A_hi, A_lo, st, num_sms); return; }
    if (variant == 1 || (variant >= 4 && variant <= 8)) {
        const int num_k = (g.K + BK - 1) / BK;
        int sp = (variant == 5 || variant == 7) ? 2 : (variant == 6 || variant == 8) ? 4 : 1;
        if (sp > num_k / 2) sp = 1;
        const int kbps = (num_k + sp - 1) / sp;
        sp = (num_k + kbps - 1) / kbps;                       // no empty K range
        if (variant == 1 || variant == 5 || variant == 6) launch<64, 8, 4>(g, A_hi, A_lo, st, num_sms, sp);
        else launch<32, 10, 5>(g, A_hi, A_lo, st, num_sms, sp);
        return;
    }
    // 128-wide tiles while they still cover half the SMs, else 64-wide ones.  The 128-wide kernel's mainloop is bound by
    // how fast L2 feeds its k-slabs (6.5-7.4 TB/s at every encoder shape, on lone CTAs), so from K = 1024 it runs in 2x2
    // clusters, which read each slab from L2 once for two tiles; a shorter K (the conv stem's 384) spends more on the
    // cluster's lockstep ring fill than it saves.  bf16x3 stays on lone CTAs.
    if (g.N >= 128 && ((g.M + BM - 1) / BM) * ((g.N + 127) / 128) >= num_sms / 2) {
        if (g.K >= 1024) launch_pp<2, 2>(g, A_hi, A_lo, st, num_sms);
        else launch_pp<1, 1>(g, A_hi, A_lo, st, num_sms);
    } else {
        // Short, narrow problems (the decoder's per-token GEMMs) cannot fill the GPU with output tiles alone and
        // a CTA walking all of K pays one TMA round trip per ring refill.  The K range is split across CTAs
        // (serial fix-up in the epilogue, see gemm_tc_kernel) until the grid covers the SMs.
        const int tiles64 = ((g.M + BM - 1) / BM) * ((g.N + 63) / 64);
        const int num_k = (g.K + BK - 1) / BK;
        int splits = 1;
        // (the fix-up is a round trip through global memory: it only pays for long K, from ~40 k-slabs, i.e. K = 5120)
        if (tiles64 < num_sms && num_k >= 40) {
            splits = num_sms / tiles64;
            if (splits > num_k / 8) splits = num_k / 8;       // at least one full ring (8 k-slabs) per split
            if (splits > 8) splits = 8;
            if (splits < 1) splits = 1;
            const int kbps = (num_k + splits - 1) / splits;
            splits = (num_k + kbps - 1) / kbps;               // no empty K range
        }
        launch<64, 8, 4>(g, A_hi, A_lo, st, num_sms, splits);
    }
}

}  // namespace wlk
