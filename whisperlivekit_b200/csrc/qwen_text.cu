// Qwen3-ASR text decoder (HF Qwen3Model + lm_head) behind the C ABI (wlk_qtext_* in include/wlk_b200.h).
//   reference third_party/qwen3-asr-causal/src/qwen3_asr_causal/model.py:
//     text model wiring :1498-1507, generate_full_hypothesis_rolling :991-1250,
//     generate_full_hypothesis_from_cached_audio :839-989, _GreedyControlSession :254-438
// The host drives the generate logic (whisperlivekit_b200/qwen_text_engine.py); this file owns the forward over a
// croppable per-session KV cache and the decode controls + argmax over the logit rows.
//
// Data layout (per round, R <= QT_ROUND_ROWS rows packed over the sessions of the call, each session's rows in position
// order, so a row always finds the keys of its predecessors either in earlier rounds or in this round's scatter):
//   residual x   fp32 [R][d];  xn act [R][d];  qkv fp32 [R][(H + 2 KV) * 128];  q act [R][H * 128];
//   K/V per session act [L][K|V][KV][max_ctx][128] (written by the QK-norm + RoPE kernel);  gate|up fp32 [R][2F]
//   hlog act [logit rows][d]: final-normed rows the lm_head runs on, in groups of logit_group rows (256 MB of fp32 logits)
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/wlk_b200.h"
#include "host.cuh"
#include "kernels.cuh"

namespace wlk {
namespace {

constexpr int QT_HD = 128;              // head_dim the kernels specialise on
constexpr int QT_ROUND_ROWS = 1024;     // rows of one forward round (workspace bound)
constexpr size_t QT_LOGIT_BYTES = (size_t)256 << 20;   // logits workspace: lm_head + pick run in groups of rows that fit
constexpr int QT_PICK_THREADS = 512;

__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    float r = 0.f;
    for (int i = 0; i < nw; ++i) r += red[i];
    return r;
}

// x[r] = embed_tokens[src] (src >= 0) or the embedding row up[-1 - src] (rows up_ld floats apart: the uploaded host rows,
// or the caller's device rows)
__global__ void qt_embed_kernel(const int32_t* __restrict__ src, const float* __restrict__ emb, const float* __restrict__ up,
                                int64_t up_ld, float* __restrict__ x, int d) {
    const int r = blockIdx.x;
    const int s = src[r];
    const float* from = s >= 0 ? emb + (int64_t)s * d : up + (int64_t)(-1 - s) * up_ld;
    for (int i = threadIdx.x; i < d; i += blockDim.x) x[(int64_t)r * d + i] = from[i];
}

// fp32 rows [R][cols] with row pitch ld -> act [R][cols] (the frame adapter's GEMM operand)
template <typename T>
__global__ void qt_rows_to_act_kernel(const float* __restrict__ in, int64_t ld, T* __restrict__ out, int cols) {
    const int r = blockIdx.x;
    for (int i = threadIdx.x; i < cols; i += blockDim.x) out[(int64_t)r * cols + i] = from_f32<T>(in[(int64_t)r * ld + i]);
}

// Qwen3RMSNorm: w * (x * rsqrt(mean(x^2) + eps)), fp32 statistics; out row = out_row ? out_row[r] : r (skip when < 0)
template <typename T>
__global__ void qt_rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, T* __restrict__ out,
                                  const int32_t* __restrict__ out_row, int d, float eps) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const int o = out_row ? out_row[r] : r;
    if (o < 0) return;
    const float* xr = x + (int64_t)r * d;
    float s = 0.f;
    for (int i = threadIdx.x; i < d; i += blockDim.x) s += xr[i] * xr[i];
    s = block_reduce_sum(s, red);
    const float inv = rsqrtf(s / (float)d + eps);
    for (int i = threadIdx.x; i < d; i += blockDim.x) out[(int64_t)o * d + i] = from_f32<T>(w[i] * (xr[i] * inv));
}

// After the fused QKV GEMM: per-head RMSNorm (q_norm / k_norm over 128 dims), HF rotate-half RoPE at the row's position,
// q -> qout [R][H*128], k / v -> the session cache.  grid (R, H + 2 KV), 128 threads (one per dim).
template <typename T>
__global__ void __launch_bounds__(QT_HD)
qt_qk_rope_kernel(const float* __restrict__ qkv, const float* __restrict__ qn, const float* __restrict__ kn,
                  const float* __restrict__ inv_freq, const int32_t* __restrict__ row_pos, const int32_t* __restrict__ row_slot,
                  void* const* __restrict__ kv_ptrs, T* __restrict__ qout, int layer, int H, int KV, int max_ctx, float eps) {
    __shared__ float red[4];
    __shared__ float vals[QT_HD];
    const int r = blockIdx.x, hh = blockIdx.y, i = threadIdx.x;
    const int W = (H + 2 * KV) * QT_HD;
    float v = qkv[(int64_t)r * W + hh * QT_HD + i];
    const int pos = row_pos[r];
    T* kvbase = reinterpret_cast<T*>(kv_ptrs[row_slot[r]]);
    if (hh >= H + KV) {                                            // v head: straight to the cache
        const int kh = hh - H - KV;
        kvbase[((((int64_t)layer * 2 + 1) * KV + kh) * max_ctx + pos) * QT_HD + i] = from_f32<T>(v);
        return;
    }
    const float s = block_reduce_sum(v * v, red);
    v = (hh < H ? qn[i] : kn[i]) * (v * rsqrtf(s / (float)QT_HD + eps));
    vals[i] = v;
    __syncthreads();
    const int j = i & (QT_HD / 2 - 1);
    const float ang = (float)pos * inv_freq[j];
    const float c = cosf(ang), sn = sinf(ang);
    const float rot = i < QT_HD / 2 ? -vals[i + QT_HD / 2] : vals[i - QT_HD / 2];
    const float o = v * c + rot * sn;
    if (hh < H) qout[(int64_t)r * H * QT_HD + hh * QT_HD + i] = from_f32<T>(o);
    else kvbase[((((int64_t)layer * 2 + 0) * KV + (hh - H)) * max_ctx + pos) * QT_HD + i] = from_f32<T>(o);
}

// fp32 mode: causal GQA attention over the session cache: the query at position p attends to cache positions 0 .. p (its own
// block's keys were scattered before this kernel).  grid (R, KV); one warp per query head of the KV group, so the
// group's heads stream the same K/V rows (L1-shared) instead of one pass per head.  Online fp32 softmax, scale 128^-0.5.
template <typename T>
__global__ void __launch_bounds__(256)
qt_attention_kernel(const T* __restrict__ q, const int32_t* __restrict__ row_pos, const int32_t* __restrict__ row_slot,
                    void* const* __restrict__ kv_ptrs, T* __restrict__ out, int layer, int H, int KV, int max_ctx) {
    __shared__ float qs[8][QT_HD];
    const int r = blockIdx.x, kh = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int G = H / KV;
    if (warp >= G) return;
    const int h = kh * G + warp;
    const int pos = row_pos[r];
    const T* kv = reinterpret_cast<const T*>(kv_ptrs[row_slot[r]]);
    const T* kb = kv + (((int64_t)layer * 2 + 0) * KV + kh) * max_ctx * QT_HD;
    const T* vb = kv + (((int64_t)layer * 2 + 1) * KV + kh) * max_ctx * QT_HD;
    const float scale = 0.08838834764831845f;                      // 128^-0.5
#pragma unroll
    for (int e = 0; e < 4; ++e) qs[warp][lane + 32 * e] = to_f32(q[(int64_t)r * H * QT_HD + h * QT_HD + lane + 32 * e]) * scale;
    __syncwarp();
    float m = -INFINITY, l = 0.f, acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = 0; k0 <= pos; k0 += 32) {
        const int k = k0 + lane;
        float sc = -INFINITY;
        if (k <= pos) {
            const T* kr = kb + (int64_t)k * QT_HD;
            float a = 0.f;
#pragma unroll 16
            for (int e = 0; e < QT_HD; ++e) a = fmaf(qs[warp][e], to_f32(kr[e]), a);
            sc = a;
        }
        const float mt = warp_max(sc);
        const float mn = fmaxf(m, mt);
        const float corr = expf(m - mn);                           // m = -inf on the first tile: corr = 0
        const float p = k <= pos ? expf(sc - mn) : 0.f;
        l = l * corr + warp_sum(p);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e] *= corr;
        const int nk = min(32, pos + 1 - k0);
        for (int j = 0; j < nk; ++j) {
            const float pj = __shfl_sync(0xffffffffu, p, j);
            const T* vr = vb + (int64_t)(k0 + j) * QT_HD;
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[e] = fmaf(pj, to_f32(vr[lane + 32 * e]), acc[e]);
        }
        m = mn;
    }
    const float inv = 1.0f / l;
#pragma unroll
    for (int e = 0; e < 4; ++e) out[(int64_t)r * H * QT_HD + h * QT_HD + lane + 32 * e] = from_f32<T>(acc[e] * inv);
}

// bf16 mode: the same attention on warp-level tensor cores (mma.sync m16n8k16, bf16 operands, fp32 accumulate).
// One CTA per (tile of <= 16 consecutive query rows of one session, KV head), one warp per query head of the group:
// the CTA stages 64-key K and V tiles in shared memory once and every head of the group runs its 16 x 64 score MMA,
// the online fp32 softmax and the P V MMA on them, so a tile's K/V leave HBM once per KV group.  Rows past n_rows of a
// tile carry zero queries and are not stored; row r attends to keys 0 .. pos0 + r.
struct QTAttnTile { int32_t row0, n_rows, slot, pos0; };
constexpr int QT_KT = 64;                         // keys per shared-memory tile
constexpr int QT_KPAD = QT_HD + 8;                // padded row: the fragment loads of a quad hit distinct banks

__device__ __forceinline__ void qt_mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t qt_pack(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t qt_pack_bf(bf16 lo, bf16 hi) {
    return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

__global__ void __launch_bounds__(256)
qt_attention_mma_kernel(const bf16* __restrict__ q, const QTAttnTile* __restrict__ tiles, void* const* __restrict__ kv_ptrs,
                        bf16* __restrict__ out, int layer, int H, int KV, int max_ctx) {
    __shared__ __align__(16) bf16 ks[QT_KT][QT_KPAD];
    __shared__ __align__(16) bf16 vs[QT_KT][QT_KPAD];
    const QTAttnTile tl = tiles[blockIdx.x];
    const int kh = blockIdx.y, G = H / KV, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int h = kh * G + warp;
    const bf16* kv = reinterpret_cast<const bf16*>(kv_ptrs[tl.slot]);
    const bf16* kb = kv + (((int64_t)layer * 2 + 0) * KV + kh) * max_ctx * QT_HD;
    const bf16* vb = kv + (((int64_t)layer * 2 + 1) * KV + kh) * max_ctx * QT_HD;
    const int kend = tl.pos0 + tl.n_rows;
    const bool ok0 = g < tl.n_rows, ok1 = g + 8 < tl.n_rows;
    const bf16* q0 = q + (int64_t)(tl.row0 + g) * H * QT_HD + h * QT_HD;
    const bf16* q1 = q + (int64_t)(tl.row0 + g + 8) * H * QT_HD + h * QT_HD;
    uint32_t qa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
        const int c = kk * 16 + 2 * t;
        qa[kk][0] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + c) : 0u;
        qa[kk][1] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + c) : 0u;
        qa[kk][2] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + c + 8) : 0u;
        qa[kk][3] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + c + 8) : 0u;
    }
    const int lim0 = min(tl.pos0 + g, kend - 1), lim1 = min(tl.pos0 + g + 8, kend - 1);
    const float scale = 0.08838834764831845f;                      // 128^-0.5
    float o[16][4];
#pragma unroll
    for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    for (int k0 = 0; k0 < kend; k0 += QT_KT) {
        __syncthreads();                                           // the previous tile is consumed
        for (int i = threadIdx.x; i < QT_KT * (QT_HD / 8); i += blockDim.x) {
            const int r = i / (QT_HD / 8), c = (i % (QT_HD / 8)) * 8;
            uint4 kz = make_uint4(0, 0, 0, 0), vz = kz;
            if (k0 + r < kend) {
                kz = *reinterpret_cast<const uint4*>(kb + (int64_t)(k0 + r) * QT_HD + c);
                vz = *reinterpret_cast<const uint4*>(vb + (int64_t)(k0 + r) * QT_HD + c);
            }
            *reinterpret_cast<uint4*>(&ks[r][c]) = kz;
            *reinterpret_cast<uint4*>(&vs[r][c]) = vz;
        }
        __syncthreads();
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&ks[8 * j + g][kk * 16 + 2 * t]);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&ks[8 * j + g][kk * 16 + 2 * t + 8]);
                qt_mma16816(s[j], qa[kk], b0, b1);
            }
        }
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = k0 + 8 * j + 2 * t + (e & 1);
                const bool ok = key <= (e < 2 ? lim0 : lim1);
                s[j][e] = ok ? s[j][e] * scale : -INFINITY;
                if (e < 2) mx0 = fmaxf(mx0, s[j][e]); else mx1 = fmaxf(mx1, s[j][e]);
            }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
        }
        const float c0 = expf(m0 - mx0), c1 = expf(m1 - mx1);     // the first tile always holds key 0: mx is finite
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = expf(s[j][0] - mx0); s[j][1] = expf(s[j][1] - mx0);
            s[j][2] = expf(s[j][2] - mx1); s[j][3] = expf(s[j][3] - mx1);
            sum0 += s[j][0] + s[j][1];
            sum1 += s[j][2] + s[j][3];
        }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
            sum0 += __shfl_xor_sync(0xffffffffu, sum0, off);
            sum1 += __shfl_xor_sync(0xffffffffu, sum1, off);
        }
        l0 = l0 * c0 + sum0;
        l1 = l1 * c1 + sum1;
#pragma unroll
        for (int n = 0; n < 16; ++n) { o[n][0] *= c0; o[n][1] *= c0; o[n][2] *= c1; o[n][3] *= c1; }
#pragma unroll
        for (int kk = 0; kk < QT_KT / 16; ++kk) {
            const uint32_t pa[4] = {qt_pack(s[2 * kk][0], s[2 * kk][1]), qt_pack(s[2 * kk][2], s[2 * kk][3]),
                                    qt_pack(s[2 * kk + 1][0], s[2 * kk + 1][1]), qt_pack(s[2 * kk + 1][2], s[2 * kk + 1][3])};
            const int kr = 16 * kk + 2 * t;
#pragma unroll
            for (int n = 0; n < 16; ++n) {
                const int c = 8 * n + g;
                const uint32_t b0 = qt_pack_bf(vs[kr][c], vs[kr + 1][c]);
                const uint32_t b1 = qt_pack_bf(vs[kr + 8][c], vs[kr + 9][c]);
                qt_mma16816(o[n], pa, b0, b1);
            }
        }
        m0 = mx0; m1 = mx1;
    }
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
    for (int n = 0; n < 16; ++n) {
        const int c = h * QT_HD + 8 * n + 2 * t;
        if (ok0) *reinterpret_cast<uint32_t*>(out + (int64_t)(tl.row0 + g) * H * QT_HD + c) = qt_pack(o[n][0] * i0, o[n][1] * i0);
        if (ok1) *reinterpret_cast<uint32_t*>(out + (int64_t)(tl.row0 + g + 8) * H * QT_HD + c) = qt_pack(o[n][2] * i1, o[n][3] * i1);
    }
}

// SwiGLU: hid[r][j] = silu(gate[r][j]) * up[r][j], gate|up = gu[r][0:F] | gu[r][F:2F] (fp32, down_proj(act(gate) * up))
template <typename T>
__global__ void qt_swiglu_kernel(const float* __restrict__ gu, T* __restrict__ hid, int rows, int F) {
    const int64_t total = (int64_t)rows * F;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / F, j = i % F;
        const float g = gu[r * 2 * F + j], u = gu[r * 2 * F + F + j];
        hid[i] = from_f32<T>(g / (1.0f + expf(-g)) * u);
    }
}

struct PickArgs {
    float* logits; int64_t ld; int vocab;
    const int32_t* hist; const int32_t* hist_off; const int32_t* hist_len;
    const int32_t* suppress; int n_suppress;
    float penalty; int penalize; int ngram; int max_consec; int wait_id;
    int32_t* picks; float* values;
};

// _GreedyControlSession.controlled_logits + argmax (model.py:335-418), one CTA per logit row, in place on the row:
// suppress (-inf) -> repetition penalty on the unique in-vocab history (first occurrence claims the token in a shared
// vocab bitmap) -> n-gram ban (finfo(float32).min) -> max-consecutive (only the wait score stays) -> argmax, lowest index on
// ties.  The modified set is a few hundred ids; the argmax then reads each logit once.
__global__ void __launch_bounds__(QT_PICK_THREADS) qt_pick_kernel(PickArgs a) {
    extern __shared__ uint32_t seen[];
    __shared__ float bv[QT_PICK_THREADS / 32];
    __shared__ int bi[QT_PICK_THREADS / 32];
    const int row = blockIdx.x, tid = threadIdx.x;
    float* lg = a.logits + (int64_t)row * a.ld;
    const int32_t* h = a.hist + a.hist_off[row];
    const int n = a.hist_len[row];
    const int words = (a.vocab + 31) / 32;
    const float fmin = -3.4028234663852886e38f;
    for (int i = tid; i < a.n_suppress; i += blockDim.x) lg[a.suppress[i]] = -INFINITY;
    for (int i = tid; i < words; i += blockDim.x) seen[i] = 0u;
    __syncthreads();
    if (a.penalize) {
        for (int i = tid; i < n; i += blockDim.x) {
            const int t = h[i];
            if (t < 0 || t >= a.vocab) continue;
            const uint32_t bit = 1u << (t & 31);
            if (atomicOr(&seen[t >> 5], bit) & bit) continue;          // not the first occurrence
            const float x = lg[t];
            lg[t] = x < 0.f ? x * a.penalty : x / a.penalty;
        }
    }
    __syncthreads();
    if (a.ngram > 0) {
        const int pre = a.ngram - 1;
        for (int s = tid; s <= n - a.ngram; s += blockDim.x) {
            bool match = true;
            for (int k = 0; k < pre && match; ++k) match = h[s + k] == h[n - pre + k];
            const int t = h[s + pre];
            if (match && t >= 0 && t < a.vocab) lg[t] = fmin;
        }
    }
    __syncthreads();
    if (a.max_consec > 0 && a.wait_id >= 0 && a.wait_id < a.vocab && n >= a.max_consec) {
        if (tid == 0) {                                               // every other entry is finfo.min
            const float w = lg[a.wait_id];
            const int pick = (w > fmin || a.wait_id == 0) ? a.wait_id : 0;
            a.picks[row] = pick;
            if (a.values) a.values[row] = pick == a.wait_id ? w : fmin;
        }
        return;
    }
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int v = tid; v < a.vocab; v += blockDim.x) {
        const float x = lg[v];
        if (x > best || (x == best && v < besti)) { best = x; besti = v; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    if ((tid & 31) == 0) { bv[tid >> 5] = best; bi[tid >> 5] = besti; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            if (bv[w] > best || (bv[w] == best && bi[w] < besti)) { best = bv[w]; besti = bi[w]; }
        if (besti == 0x7fffffff) besti = 0;                            // NaN row: torch.argmax would say 0 too
        a.picks[row] = besti;
        if (a.values) a.values[row] = best;
    }
}

struct QTLayerW {
    void *Wqkv = nullptr, *Wo = nullptr, *Wgu = nullptr, *Wd = nullptr;
    float *qn = nullptr, *kn = nullptr, *ln1 = nullptr, *ln2 = nullptr;
};

struct QTSession {
    bool open = false;
    int len = 0;
    void* kv = nullptr;
};

// QwenAudioSurgeryFrameAdapter (reference model.py:631-691): proj [d][in_dim] without bias, then `nb` blocks of
// x + scale * down(silu(gate(n)) * up(n)), n = RMSNorm(x) with eps 1e-6 (the reference's own RMSNorm, model.py:83-91).
// Tensors are stashed on load and packed by finalize, which derives in_dim, nb and the hidden width from their shapes.
struct QTAdapter {
    int in_dim = 0, hidden = 0, nb = 0;
    float scale = 0.f;
    void* Wp = nullptr;                              // act [d][in_dim]
    std::vector<float*> norm;                        // fp32 [d]
    std::vector<void*> Wgu, Wd;                      // act [2 hidden][d] (gate | up), [d][hidden]
    void* a_in = nullptr;                            // act [QT_ROUND_ROWS][in_dim]
    float* a_gu = nullptr;                           // fp32 [QT_ROUND_ROWS][2 hidden]
    void* a_hid = nullptr;                           // act [QT_ROUND_ROWS][hidden]
};
constexpr float QT_ADAPTER_EPS = 1e-6f;

}  // namespace
}  // namespace wlk

using namespace wlk;

struct wlk_qtext {
    wlk_qtext_dims dims{};
    wlk_config cfg{};
    int act = DT_F32, gemm_backend = WLK_BACKEND_SIMT, num_sms = 132;
    cudaStream_t st = nullptr;
    std::mutex mu;
    DeviceAllocs allocs;
    size_t bytes_weights = 0, bytes_sessions = 0, bytes_workspace = 0, kv_bytes = 0;
    float *emb = nullptr, *normw = nullptr, *inv_freq = nullptr;
    void* head = nullptr;                               // lm_head [V][d] act type (the embedding table when tied)
    std::vector<QTLayerW> L;
    std::set<std::string> loaded;
    bool finalized = false;
    WeightUpload upload;
    std::vector<QTSession> sess;
    float *x = nullptr, *qkv = nullptr, *gu = nullptr, *up = nullptr, *logits = nullptr, *values_d = nullptr;
    void *xn = nullptr, *qb = nullptr, *att = nullptr, *hid = nullptr, *hlog = nullptr;
    int32_t* picks_d = nullptr;
    float* up_h = nullptr;                               // pinned: the round's host embedding rows, one H2D copy per round
    cudaEvent_t stg_ev = nullptr;                        // recorded after the last H2D copy out of stg_h / up_h
    int32_t* pick_d = nullptr; size_t pick_cap = 0;      // device copy of a pick call's histories, suppress list, offsets
    int logit_group = 0;
    int up_rows = 0;                                     // rows of `up` (uploaded embedding rows)
    int logit_cap = 0, n_logit = 0;                      // rows of hlog; rows the last forward kept
    float* sk_scratch = nullptr; int* sk_counters = nullptr;
    uint8_t *stg_h = nullptr, *stg_d = nullptr; size_t stg_bytes = 0;
    std::map<std::string, std::pair<std::vector<int64_t>, std::vector<float>>> adapter_stash;   // until finalize
    bool has_adapter = false;
    QTAdapter ad;
    size_t es() const { return dtype_size(act); }
};

namespace {

void tgemm(wlk_qtext* t, GemmArgs& g) {
    if (g.M <= 0) return;
    g.sk_scratch = t->sk_scratch; g.sk_scratch_floats = SK_SCRATCH_FLOATS;
    g.sk_counters = t->sk_counters; g.sk_max_tiles = SK_MAX_TILES;
    if (t->gemm_backend == WLK_BACKEND_TCGEN05) {
        std::string why;
        WLK_CHECK(gemm_tcgen05_supported(g, &why), "text decoder GEMM %dx%dx%d has no wgmma kernel: %s", g.M, g.N, g.K, why.c_str());
        gemm_tcgen05(g, t->st, t->num_sms);
    } else {
        gemm_simt(g, t->st);
    }
}

void load_tensor(wlk_qtext* t, const std::string& name, const float* host, const int64_t* shape, int ndim) {
    const wlk_qtext_dims& D = t->dims;
    const int d = D.d_model, F = D.ffn_dim, qd = D.n_head * QT_HD, kvd = D.n_kv_head * QT_HD;
    const int64_t n = numel(shape, ndim);
    const size_t es = t->es();
    auto mat = [&](void* dst, int64_t rows, int64_t cols) { expect_shape(name.c_str(), shape, ndim, {rows, cols}); t->upload.put(host, n, dst, t->act, t->st); };
    auto vec = [&](float* dst, int64_t len) { expect_shape(name.c_str(), shape, ndim, {len}); t->upload.put(host, n, dst, DT_F32, t->st); };
    if (name == "embed_tokens.weight") {
        expect_shape(name.c_str(), shape, ndim, {D.vocab, d});
        t->upload.put(host, n, t->emb, DT_F32, t->st);
        if (D.tied) t->upload.put(host, n, t->head, t->act, t->st);
    }
    else if (name == "lm_head.weight") { WLK_CHECK(!D.tied, "this geometry ties lm_head to embed_tokens"); mat(t->head, D.vocab, d); }
    else if (name == "norm.weight") vec(t->normw, d);
    else if (name == "rotary_emb.inv_freq") vec(t->inv_freq, QT_HD / 2);     // optional: the host's own RoPE frequencies
    else if (name.rfind("adapter.", 0) == 0) {                                   // optional: the frame adapter, packed by finalize
        WLK_CHECK(!t->finalized, "adapter tensor %s loaded after finalize", name.c_str());
        t->adapter_stash[name] = {std::vector<int64_t>(shape, shape + ndim), std::vector<float>(host, host + n)};
    }
    else if (name.rfind("layers.", 0) == 0) {
        const size_t dot = name.find('.', 7);
        WLK_CHECK(dot != std::string::npos, "unknown tensor %s", name.c_str());
        const int li = atoi(name.substr(7, dot - 7).c_str());
        WLK_CHECK(li >= 0 && li < D.n_layer, "layer index out of range in %s", name.c_str());
        const std::string rest = name.substr(dot + 1);
        QTLayerW& Lw = t->L[li];
        if (rest == "self_attn.q_proj.weight") { expect_shape(name.c_str(), shape, ndim, {qd, d}); t->upload.put(host, n, Lw.Wqkv, t->act, t->st); }
        else if (rest == "self_attn.k_proj.weight") { expect_shape(name.c_str(), shape, ndim, {kvd, d}); t->upload.put(host, n, (char*)Lw.Wqkv + (size_t)qd * d * es, t->act, t->st); }
        else if (rest == "self_attn.v_proj.weight") { expect_shape(name.c_str(), shape, ndim, {kvd, d}); t->upload.put(host, n, (char*)Lw.Wqkv + (size_t)(qd + kvd) * d * es, t->act, t->st); }
        else if (rest == "self_attn.o_proj.weight") mat(Lw.Wo, d, qd);
        else if (rest == "self_attn.q_norm.weight") vec(Lw.qn, QT_HD);
        else if (rest == "self_attn.k_norm.weight") vec(Lw.kn, QT_HD);
        else if (rest == "mlp.gate_proj.weight") { expect_shape(name.c_str(), shape, ndim, {F, d}); t->upload.put(host, n, Lw.Wgu, t->act, t->st); }
        else if (rest == "mlp.up_proj.weight") { expect_shape(name.c_str(), shape, ndim, {F, d}); t->upload.put(host, n, (char*)Lw.Wgu + (size_t)F * d * es, t->act, t->st); }
        else if (rest == "mlp.down_proj.weight") mat(Lw.Wd, d, F);
        else if (rest == "input_layernorm.weight") vec(Lw.ln1, d);
        else if (rest == "post_attention_layernorm.weight") vec(Lw.ln2, d);
        else WLK_CHECK(false, "unknown tensor %s", name.c_str());
    }
    else WLK_CHECK(false, "unknown tensor %s", name.c_str());
    t->loaded.insert(name);
}

std::vector<std::string> required(const wlk_qtext_dims& D) {
    std::vector<std::string> r = {"embed_tokens.weight", "norm.weight"};
    if (!D.tied) r.push_back("lm_head.weight");
    for (int i = 0; i < D.n_layer; ++i) {
        const std::string p = "layers." + std::to_string(i) + ".";
        for (const char* s : {"self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "self_attn.q_norm",
                              "self_attn.k_norm", "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj", "input_layernorm",
                              "post_attention_layernorm"})
            r.push_back(p + s + ".weight");
    }
    return r;
}

// Pack the stashed adapter tensors (no-op when none were loaded).
void build_adapter(wlk_qtext* t) {
    auto& st = t->adapter_stash;
    if (st.empty()) return;
    const int d = t->dims.d_model;
    auto get = [&](const std::string& name) -> std::pair<std::vector<int64_t>, std::vector<float>>& {
        auto it = st.find(name);
        WLK_CHECK(it != st.end(), "adapter tensor %s missing", name.c_str());
        return it->second;
    };
    auto& proj = get("adapter.proj.weight");
    WLK_CHECK(proj.first.size() == 2 && proj.first[0] == d && proj.first[1] >= 8 && proj.first[1] % 8 == 0,
              "adapter.proj.weight must be [d_model][in_dim] with in_dim a multiple of 8");
    QTAdapter& A = t->ad;
    A.in_dim = (int)proj.first[1];
    int nb = 0;
    while (st.count("adapter.blocks." + std::to_string(nb) + ".norm.weight")) ++nb;
    A.nb = nb;
    size_t used = 1;
    if (nb > 0) {
        auto& rs = get("adapter.residual_scale");
        WLK_CHECK(rs.second.size() == 1, "adapter.residual_scale must hold one value");
        A.scale = rs.second[0];
        used++;
        A.hidden = (int)get("adapter.blocks.0.mlp.gate.weight").first[0];
        WLK_CHECK(A.hidden >= 8 && A.hidden % 8 == 0, "adapter hidden width %d must be a positive multiple of 8", A.hidden);
    } else if (st.count("adapter.residual_scale")) {
        used++;
    }
    const size_t es = t->es();
    size_t* aw = &t->bytes_weights;
    A.Wp = t->allocs.take((size_t)d * A.in_dim * es, aw);
    t->upload.put(proj.second.data(), proj.second.size(), A.Wp, t->act, t->st);
    const int64_t H = A.hidden;
    for (int i = 0; i < nb; ++i) {
        const std::string p = "adapter.blocks." + std::to_string(i) + ".";
        auto& nw = get(p + "norm.weight");
        auto& g = get(p + "mlp.gate.weight");
        auto& u = get(p + "mlp.up.weight");
        auto& dn = get(p + "mlp.down.weight");
        WLK_CHECK(nw.first == std::vector<int64_t>{d}, "%snorm.weight must be [d_model]", p.c_str());
        WLK_CHECK(g.first == (std::vector<int64_t>{H, d}) && u.first == (std::vector<int64_t>{H, d}),
                  "%smlp.gate / mlp.up must be [hidden][d_model] with the hidden width of block 0", p.c_str());
        WLK_CHECK(dn.first == (std::vector<int64_t>{d, H}), "%smlp.down.weight must be [d_model][hidden]", p.c_str());
        float* nd = (float*)t->allocs.take((size_t)d * 4, aw);
        t->upload.put(nw.second.data(), nw.second.size(), nd, DT_F32, t->st);
        void* gu = t->allocs.take((size_t)2 * H * d * es, aw);
        t->upload.put(g.second.data(), g.second.size(), gu, t->act, t->st);
        t->upload.put(u.second.data(), u.second.size(), (char*)gu + (size_t)H * d * es, t->act, t->st);
        void* wd = t->allocs.take((size_t)d * H * es, aw);
        t->upload.put(dn.second.data(), dn.second.size(), wd, t->act, t->st);
        A.norm.push_back(nd); A.Wgu.push_back(gu); A.Wd.push_back(wd);
        used += 4;
    }
    WLK_CHECK(used == st.size(), "%zu adapter tensors do not belong to an adapter of %d blocks", st.size() - used, nb);
    size_t* ws = &t->bytes_workspace;
    A.a_in = t->allocs.take((size_t)QT_ROUND_ROWS * A.in_dim * es, ws);
    if (nb > 0) {
        A.a_gu = (float*)t->allocs.take((size_t)QT_ROUND_ROWS * 2 * H * 4, ws);
        A.a_hid = t->allocs.take((size_t)QT_ROUND_ROWS * H * es, ws);
    }
    st.clear();
    t->has_adapter = true;
}

void create(const wlk_qtext_dims* dims, const wlk_config* cfg, wlk_qtext** out) {
    WLK_CHECK(dims && cfg && out, "null argument");
    const wlk_qtext_dims& D = *dims;
    WLK_CHECK(D.head_dim == QT_HD, "head_dim must be %d", QT_HD);
    WLK_CHECK(D.n_kv_head >= 1 && D.n_head % D.n_kv_head == 0 && D.n_head / D.n_kv_head <= 8, "n_head must be a multiple (<= 8x) of n_kv_head");
    WLK_CHECK(D.d_model % 8 == 0 && D.ffn_dim % 8 == 0 && D.vocab >= 1, "d_model and ffn_dim must be multiples of 8");
    WLK_CHECK(D.max_ctx >= 1 && D.max_ctx <= 32768, "max_ctx must be in [1, 32768]");
    WLK_CHECK((size_t)(D.vocab + 31) / 32 * 4 <= 200 * 1024, "vocab too large for the pick kernel's bitmap");
    WLK_CHECK(cfg->max_sessions >= 1 && cfg->max_batch >= 1, "max_sessions / max_batch must be >= 1");
    const int num_sms = open_sm90_device(cfg->device);

    auto* t = new wlk_qtext();
    t->dims = D; t->cfg = *cfg;
    t->num_sms = num_sms;
    t->act = cfg->precision == WLK_PREC_BF16 ? DT_BF16 : DT_F32;
    t->gemm_backend = t->act == DT_BF16 ? WLK_BACKEND_TCGEN05 : WLK_BACKEND_SIMT;
    CUDA_CHECK(cudaStreamCreateWithFlags(&t->st, cudaStreamNonBlocking));
    const size_t es = t->es();
    const int d = D.d_model, F = D.ffn_dim, H = D.n_head, KV = D.n_kv_head;
    const size_t W = (size_t)(H + 2 * KV) * QT_HD;
    size_t* aw = &t->bytes_weights;
    t->emb = (float*)t->allocs.take((size_t)D.vocab * d * 4, aw);
    t->head = t->allocs.take((size_t)D.vocab * d * es, aw);
    t->normw = (float*)t->allocs.take((size_t)d * 4, aw);
    t->inv_freq = (float*)t->allocs.take(QT_HD / 2 * 4, aw);
    t->L.resize(D.n_layer);
    for (auto& Lw : t->L) {
        Lw.Wqkv = t->allocs.take(W * d * es, aw);
        Lw.Wo = t->allocs.take((size_t)d * H * QT_HD * es, aw);
        Lw.Wgu = t->allocs.take((size_t)2 * F * d * es, aw);
        Lw.Wd = t->allocs.take((size_t)d * F * es, aw);
        Lw.qn = (float*)t->allocs.take(QT_HD * 4, aw); Lw.kn = (float*)t->allocs.take(QT_HD * 4, aw);
        Lw.ln1 = (float*)t->allocs.take((size_t)d * 4, aw); Lw.ln2 = (float*)t->allocs.take((size_t)d * 4, aw);
    }
    {   // default inv_freq = 1 / theta^(2i / 128) in fp32 arithmetic like HF's default rope init (fp32 exponent, pow, then
        // 1 / x); libm's powf can still land one ulp away from torch's pow in a few entries, so hosts load
        // "rotary_emb.inv_freq" (whisperlivekit_b200/qwen_text_engine.py always does)
        std::vector<float> f(QT_HD / 2);
        for (int i = 0; i < QT_HD / 2; ++i) f[i] = 1.0f / powf(D.rope_theta, (float)(2 * i) / (float)QT_HD);
        CUDA_CHECK(cudaMemcpy(t->inv_freq, f.data(), f.size() * 4, cudaMemcpyHostToDevice));
    }
    const size_t R = QT_ROUND_ROWS;
    size_t* ws = &t->bytes_workspace;
    t->x = (float*)t->allocs.take(R * d * 4, ws);
    t->xn = t->allocs.take(R * d * es, ws);
    t->qkv = (float*)t->allocs.take(R * W * 4, ws);
    t->qb = t->allocs.take(R * H * QT_HD * es, ws);
    t->att = t->allocs.take(R * H * QT_HD * es, ws);
    t->gu = (float*)t->allocs.take(R * 2 * F * 4, ws);
    t->hid = t->allocs.take(R * F * es, ws);
    t->up_rows = (int)R;
    t->up = (float*)t->allocs.take(R * d * 4, ws);
    t->logit_cap = cfg->max_batch * 288;
    t->hlog = t->allocs.take((size_t)t->logit_cap * d * es, ws);
    t->logit_group = (int)std::max<size_t>(1, std::min<size_t>((size_t)t->logit_cap, QT_LOGIT_BYTES / ((size_t)D.vocab * 4)));
    t->logits = (float*)t->allocs.take((size_t)t->logit_group * D.vocab * 4, ws);
    t->picks_d = (int32_t*)t->allocs.take((size_t)t->logit_cap * 4, ws);
    t->values_d = (float*)t->allocs.take((size_t)t->logit_cap * 4, ws);
    if (t->gemm_backend == WLK_BACKEND_TCGEN05) {
        t->sk_scratch = (float*)t->allocs.take(SK_SCRATCH_FLOATS * 4, ws);
        t->sk_counters = (int*)t->allocs.take(SK_MAX_TILES * 4, ws);
    }
    t->stg_bytes = R * 32 + (size_t)cfg->max_batch * 16 + 8192;
    CUDA_CHECK(cudaMallocHost(&t->stg_h, t->stg_bytes));
    CUDA_CHECK(cudaMallocHost(&t->up_h, R * d * 4));
    CUDA_CHECK(cudaEventCreateWithFlags(&t->stg_ev, cudaEventDisableTiming));
    t->stg_d = (uint8_t*)t->allocs.take(t->stg_bytes, ws);
    t->kv_bytes = (size_t)D.n_layer * 2 * KV * D.max_ctx * QT_HD * es;
    t->sess.resize(cfg->max_sessions);
    CUDA_CHECK(cudaFuncSetAttribute(qt_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    *out = t;
}

void destroy(wlk_qtext* t) {
    cudaStreamSynchronize(t->st);
    for (auto& s : t->sess) if (s.kv) cudaFree(s.kv);
    t->allocs.free_all();
    t->upload.release();
    if (t->stg_h) cudaFreeHost(t->stg_h);
    if (t->up_h) cudaFreeHost(t->up_h);
    if (t->pick_d) cudaFree(t->pick_d);
    if (t->stg_ev) cudaEventDestroy(t->stg_ev);
    cudaStreamDestroy(t->st);
    delete t;
}

QTSession& tsession(wlk_qtext* t, int32_t sid) {
    WLK_CHECK(sid >= 0 && sid < (int)t->sess.size() && t->sess[sid].open, "invalid session id %d", sid);
    return t->sess[sid];
}

// Attention tiles of one round (the bf16 kernel's CTAs): <= 16 consecutive rows of one slot, a new tile whenever the
// slot changes.  Rows of a slot are contiguous and at consecutive positions, so a tile's row k sits at pos0 + k.
int make_tiles(const int32_t* pos, const int32_t* slot, int R, QTAttnTile* tiles) {
    int n = 0;
    for (int k = 0; k < R; ++k) {
        if (n == 0 || tiles[n - 1].slot != slot[k] || tiles[n - 1].n_rows == 16) tiles[n++] = QTAttnTile{k, 0, slot[k], pos[k]};
        tiles[n - 1].n_rows++;
    }
    return n;
}

// The per-kernel launches of a round, shared by run_round and the op-level entry points.
template <typename T>
void launch_rmsnorm(wlk_qtext* t, const float* x, const float* w, void* out, const int32_t* out_row_d, int R, float eps) {
    qt_rmsnorm_kernel<T><<<R, 256, 0, t->st>>>(x, w, (T*)out, out_row_d, t->dims.d_model, eps);
}

template <typename T>
void launch_qk_rope(wlk_qtext* t, const float* qkv, const float* qn, const float* kn, const int32_t* pos_d, const int32_t* slot_d,
                    void* const* kv_d, int layer, void* qout, int R) {
    const wlk_qtext_dims& D = t->dims;
    qt_qk_rope_kernel<T><<<dim3(R, D.n_head + 2 * D.n_kv_head), QT_HD, 0, t->st>>>(qkv, qn, kn, t->inv_freq, pos_d, slot_d, kv_d,
                                                                                 (T*)qout, layer, D.n_head, D.n_kv_head,
                                                                                 D.max_ctx, D.rms_eps);
}

template <typename T>
void launch_attention(wlk_qtext* t, const void* q, const int32_t* pos_d, const int32_t* slot_d, void* const* kv_d,
                      const QTAttnTile* tiles_d, int n_tiles, int layer, void* out, int R) {
    const int H = t->dims.n_head, KV = t->dims.n_kv_head;
    if (t->act == DT_BF16)
        qt_attention_mma_kernel<<<dim3(n_tiles, KV), 32 * (H / KV), 0, t->st>>>((const bf16*)q, tiles_d, kv_d, (bf16*)out,
                                                                              layer, H, KV, t->dims.max_ctx);
    else
        qt_attention_kernel<T><<<dim3(R, KV), 32 * (H / KV), 0, t->st>>>((const T*)q, pos_d, slot_d, kv_d, (T*)out, layer,
                                                                        H, KV, t->dims.max_ctx);
}

template <typename T>
void launch_swiglu(wlk_qtext* t, const float* gu, void* hid, int R, int F) {
    const int64_t total = (int64_t)R * F;
    const int blocks = (int)std::min<int64_t>((total + 255) / 256, 65535);
    qt_swiglu_kernel<T><<<blocks, 256, 0, t->st>>>(gu, (T*)hid, R, F);
}

template <typename T>
void run_round(wlk_qtext* t, int R, const int32_t* src_d, const int32_t* pos_d, const int32_t* slot_d, void* const* kv_d,
               const int32_t* logit_row_d, const QTAttnTile* tiles_d, int n_tiles, const float* up, int64_t up_ld) {
    const wlk_qtext_dims& D = t->dims;
    const int d = D.d_model, F = D.ffn_dim, H = D.n_head, KV = D.n_kv_head;
    const int W = (H + 2 * KV) * QT_HD;
    qt_embed_kernel<<<R, 256, 0, t->st>>>(src_d, t->emb, up, up_ld, t->x, d);
    for (int li = 0; li < D.n_layer; ++li) {
        QTLayerW& Lw = t->L[li];
        launch_rmsnorm<T>(t, t->x, Lw.ln1, t->xn, nullptr, R, D.rms_eps);
        {   GemmArgs g;
            g.A = t->xn; g.a_type = t->act; g.lda = d; g.W = Lw.Wqkv; g.w_type = t->act; g.ldw = d;
            g.M = R; g.N = W; g.K = d;
            g.epi.C = t->qkv; g.epi.c_type = DT_F32; g.epi.ldc = W;
            tgemm(t, g); }
        launch_qk_rope<T>(t, t->qkv, Lw.qn, Lw.kn, pos_d, slot_d, kv_d, li, t->qb, R);
        launch_attention<T>(t, t->qb, pos_d, slot_d, kv_d, tiles_d, n_tiles, li, t->att, R);
        {   GemmArgs g;
            g.A = t->att; g.a_type = t->act; g.lda = H * QT_HD; g.W = Lw.Wo; g.w_type = t->act; g.ldw = H * QT_HD;
            g.M = R; g.N = d; g.K = H * QT_HD;
            g.epi.residual = t->x; g.epi.ldr = d; g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            tgemm(t, g); }
        launch_rmsnorm<T>(t, t->x, Lw.ln2, t->xn, nullptr, R, D.rms_eps);
        {   GemmArgs g;
            g.A = t->xn; g.a_type = t->act; g.lda = d; g.W = Lw.Wgu; g.w_type = t->act; g.ldw = d;
            g.M = R; g.N = 2 * F; g.K = d;
            g.epi.C = t->gu; g.epi.c_type = DT_F32; g.epi.ldc = 2 * F;
            tgemm(t, g); }
        launch_swiglu<T>(t, t->gu, t->hid, R, F);
        {   GemmArgs g;
            g.A = t->hid; g.a_type = t->act; g.lda = F; g.W = Lw.Wd; g.w_type = t->act; g.ldw = F;
            g.M = R; g.N = d; g.K = F;
            g.epi.residual = t->x; g.epi.ldr = d; g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            tgemm(t, g); }
    }
    launch_rmsnorm<T>(t, t->x, t->normw, t->hlog, logit_row_d, R, D.rms_eps);
    CUDA_CHECK(cudaGetLastError());
}

// embeds: host rows [n_embeds][d_model] (staged through pinned memory), or, when embeds_ld > 0, device rows embeds_ld
// floats apart that the embedding gather reads in place.
void forward(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_off, const float* embeds,
             int n_embeds, const int32_t* logit_rows, int64_t embeds_ld = 0) {
    const wlk_qtext_dims& D = t->dims;
    const bool dev_rows = embeds_ld > 0;
    WLK_CHECK(t->finalized, "weights not finalized");
    WLK_CHECK(n >= 1 && n <= t->cfg.max_batch, "batch %d outside [1, %d]", n, t->cfg.max_batch);
    int n_logit = 0;
    for (int i = 0; i < n; ++i) {
        QTSession& s = tsession(t, sids[i]);
        for (int j = 0; j < i; ++j) WLK_CHECK(sids[j] != sids[i], "session %d appears twice in the batch", sids[i]);
        const int r = row_off[i + 1] - row_off[i];
        WLK_CHECK(r >= 1, "session %d has no rows", sids[i]);
        WLK_CHECK(s.len + r <= D.max_ctx, "context full: session %d holds %d positions, %d more exceed max_ctx %d", sids[i], s.len, r, D.max_ctx);
        WLK_CHECK(logit_rows[i] >= 0 && logit_rows[i] <= r, "logit_rows[%d] = %d outside [0, %d]", i, logit_rows[i], r);
        n_logit += logit_rows[i];
    }
    WLK_CHECK(n_logit <= t->logit_cap, "%d logit rows exceed the engine's %d", n_logit, t->logit_cap);
    const int total = row_off[n] - row_off[0];
    for (int r = 0; r < total; ++r) {
        const int s = row_src[row_off[0] + r];
        WLK_CHECK(s < D.vocab && (s >= 0 || -1 - s < n_embeds), "row %d: source %d is neither a token id nor an embedding row", r, s);
    }
    // the packed row list: (session index, position, logit row or -1)
    std::vector<int> r_sess(total), r_pos(total), r_log(total);
    {   int r = 0, lg = 0;
        for (int i = 0; i < n; ++i) {
            const int cnt = row_off[i + 1] - row_off[i];
            for (int k = 0; k < cnt; ++k, ++r) {
                r_sess[r] = i; r_pos[r] = t->sess[sids[i]].len + k;
                r_log[r] = k >= cnt - logit_rows[i] ? lg++ : -1;
            }
        }
    }
    for (int r0 = 0; r0 < total; r0 += QT_ROUND_ROWS) {
        const int R = std::min(QT_ROUND_ROWS, total - r0);
        size_t off = 0;
        auto carve = [&](size_t bytes) { size_t o = (off + 255) / 256 * 256; off = o + bytes; WLK_CHECK(off <= t->stg_bytes, "staging overflow"); return o; };
        const size_t o_src = carve((size_t)R * 4), o_pos = carve((size_t)R * 4), o_slot = carve((size_t)R * 4),
                     o_log = carve((size_t)R * 4), o_kv = carve((size_t)n * sizeof(void*)),
                     o_tile = carve((size_t)R * sizeof(QTAttnTile));
        CUDA_CHECK(cudaEventSynchronize(t->stg_ev));     // the previous H2D copy out of stg_h / up_h has been consumed
        int32_t* src = reinterpret_cast<int32_t*>(t->stg_h + o_src);
        int32_t* pos = reinterpret_cast<int32_t*>(t->stg_h + o_pos);
        int32_t* slot = reinterpret_cast<int32_t*>(t->stg_h + o_slot);
        int32_t* lrow = reinterpret_cast<int32_t*>(t->stg_h + o_log);
        void** kvp = reinterpret_cast<void**>(t->stg_h + o_kv);
        for (int i = 0; i < n; ++i) kvp[i] = t->sess[sids[i]].kv;
        // embedding rows of this round go to `up` in the order they appear: packed into pinned memory, one copy
        int n_up = 0;
        for (int k = 0; k < R; ++k) {
            const int r = r0 + k;
            int s = row_src[row_off[0] + r];
            if (s < 0 && !dev_rows) {
                memcpy(t->up_h + (size_t)n_up * D.d_model, embeds + (size_t)(-1 - s) * D.d_model, (size_t)D.d_model * 4);
                s = -1 - n_up++;
            }
            src[k] = s; pos[k] = r_pos[r]; slot[k] = r_sess[r]; lrow[k] = r_log[r];
        }
        QTAttnTile* tiles = reinterpret_cast<QTAttnTile*>(t->stg_h + o_tile);
        const int n_tiles = make_tiles(pos, slot, R, tiles);
        if (n_up) CUDA_CHECK(cudaMemcpyAsync(t->up, t->up_h, (size_t)n_up * D.d_model * 4, cudaMemcpyHostToDevice, t->st));
        CUDA_CHECK(cudaMemcpyAsync(t->stg_d, t->stg_h, off, cudaMemcpyHostToDevice, t->st));
        CUDA_CHECK(cudaEventRecord(t->stg_ev, t->st));
        const int32_t* src_d = reinterpret_cast<const int32_t*>(t->stg_d + o_src);
        const int32_t* pos_d = reinterpret_cast<const int32_t*>(t->stg_d + o_pos);
        const int32_t* slot_d = reinterpret_cast<const int32_t*>(t->stg_d + o_slot);
        const int32_t* log_d = reinterpret_cast<const int32_t*>(t->stg_d + o_log);
        void* const* kv_d = reinterpret_cast<void* const*>(t->stg_d + o_kv);
        const QTAttnTile* tiles_d = reinterpret_cast<const QTAttnTile*>(t->stg_d + o_tile);
        const float* up = dev_rows ? embeds : t->up;
        const int64_t up_ld = dev_rows ? embeds_ld : D.d_model;
        if (t->act == DT_F32) run_round<float>(t, R, src_d, pos_d, slot_d, kv_d, log_d, tiles_d, n_tiles, up, up_ld);
        else run_round<bf16>(t, R, src_d, pos_d, slot_d, kv_d, log_d, tiles_d, n_tiles, up, up_ld);
    }
    // no host sync here: the pick (or logits) call that follows synchronizes once for the whole phase
    for (int i = 0; i < n; ++i) t->sess[sids[i]].len += row_off[i + 1] - row_off[i];
    t->n_logit = n_logit;
}

void head_group(wlk_qtext* t, int row0, int rows) {
    GemmArgs g;
    g.A = (const char*)t->hlog + (size_t)row0 * t->dims.d_model * t->es(); g.a_type = t->act; g.lda = t->dims.d_model;
    g.W = t->head; g.w_type = t->act; g.ldw = t->dims.d_model;
    g.M = rows; g.N = t->dims.vocab; g.K = t->dims.d_model;
    g.epi.C = t->logits; g.epi.c_type = DT_F32; g.epi.ldc = t->dims.vocab;
    tgemm(t, g);
}

void pick(wlk_qtext* t, const int32_t* hist, int n_hist, const int32_t* hist_off, const int32_t* hist_len, const int32_t* suppress,
          int n_suppress, float penalty, int ngram, int max_consec, int wait_id, int32_t* picks, float* values) {
    const wlk_qtext_dims& D = t->dims;
    WLK_CHECK(t->finalized, "weights not finalized");
    const int N = t->n_logit;
    if (N == 0) return;
    for (int j = 0; j < N; ++j)
        WLK_CHECK(hist_off[j] >= 0 && hist_len[j] >= 0 && hist_off[j] + hist_len[j] <= n_hist, "history of row %d out of range", j);
    std::vector<int32_t> sup;
    for (int i = 0; i < n_suppress; ++i) if (suppress[i] >= 0 && suppress[i] < D.vocab) sup.push_back(suppress[i]);
    // the reference only arms max-consecutive when the wait token is not suppressed (model.py:1067-1072)
    for (int32_t v : sup) if (v == wait_id) wait_id = -1;
    // one device buffer, grown on demand: [2N offsets/lengths][suppress][histories]
    const size_t need = (size_t)2 * N + sup.size() + (size_t)n_hist + 1;
    if (need > t->pick_cap) {
        CUDA_CHECK(cudaStreamSynchronize(t->st));
        if (t->pick_d) CUDA_CHECK(cudaFree(t->pick_d));
        t->pick_cap = std::max(need, (size_t)1 << 16);
        CUDA_CHECK(cudaMalloc(&t->pick_d, t->pick_cap * 4));
    }
    int32_t* meta_d = t->pick_d;
    int32_t* hist_d = t->pick_d + 2 * N + sup.size();
    if (n_hist) CUDA_CHECK(cudaMemcpyAsync(hist_d, hist, (size_t)n_hist * 4, cudaMemcpyHostToDevice, t->st));
    CUDA_CHECK(cudaMemcpyAsync(meta_d, hist_off, (size_t)N * 4, cudaMemcpyHostToDevice, t->st));
    CUDA_CHECK(cudaMemcpyAsync(meta_d + N, hist_len, (size_t)N * 4, cudaMemcpyHostToDevice, t->st));
    if (!sup.empty()) CUDA_CHECK(cudaMemcpyAsync(meta_d + 2 * N, sup.data(), sup.size() * 4, cudaMemcpyHostToDevice, t->st));
    const size_t smem = (size_t)(D.vocab + 31) / 32 * 4;
    for (int g0 = 0; g0 < N; g0 += t->logit_group) {
        const int rows = std::min(t->logit_group, N - g0);
        head_group(t, g0, rows);
        PickArgs a;
        a.logits = t->logits; a.ld = D.vocab; a.vocab = D.vocab;
        a.hist = hist_d; a.hist_off = meta_d + g0; a.hist_len = meta_d + N + g0;
        a.suppress = meta_d + 2 * N; a.n_suppress = (int)sup.size();
        a.penalty = penalty; a.penalize = penalty != 1.0f && penalty > 0.0f; a.ngram = ngram; a.max_consec = max_consec;
        a.wait_id = wait_id; a.picks = t->picks_d + g0; a.values = t->values_d + g0;
        qt_pick_kernel<<<rows, QT_PICK_THREADS, smem, t->st>>>(a);
        CUDA_CHECK(cudaGetLastError());
    }
    CUDA_CHECK(cudaMemcpyAsync(picks, t->picks_d, (size_t)N * 4, cudaMemcpyDeviceToHost, t->st));
    if (values) CUDA_CHECK(cudaMemcpyAsync(values, t->values_d, (size_t)N * 4, cudaMemcpyDeviceToHost, t->st));
    CUDA_CHECK(cudaStreamSynchronize(t->st));            // the one host sync of a forward + pick phase
}

void logits_out(wlk_qtext* t, int row0, int rows, float* out) {
    WLK_CHECK(t->finalized, "weights not finalized");
    WLK_CHECK(row0 >= 0 && rows >= 0 && row0 + rows <= t->n_logit, "logit rows [%d, %d) outside the last forward's %d", row0, row0 + rows, t->n_logit);
    for (int g0 = 0; g0 < rows; g0 += t->logit_group) {
        const int r = std::min(t->logit_group, rows - g0);
        head_group(t, row0 + g0, r);
        CUDA_CHECK(cudaMemcpyAsync(out + (size_t)g0 * t->dims.vocab, t->logits, (size_t)r * t->dims.vocab * 4, cudaMemcpyDeviceToHost, t->st));
        CUDA_CHECK(cudaStreamSynchronize(t->st));
    }
}

// ---- op-level entry points: one kernel of a round on caller-owned device buffers ----------------------------------
// Device copies of an op call's host index arrays, freed once the op's work on the stream is done.
struct OpUpload {
    wlk_qtext* t;
    std::vector<void*> bufs;
    template <typename X>
    const X* put(const X* host, size_t n) {
        void* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(X)));
        bufs.push_back(p);
        CUDA_CHECK(cudaMemcpyAsync(p, host, n * sizeof(X), cudaMemcpyHostToDevice, t->st));
        return (const X*)p;
    }
    ~OpUpload() {
        cudaStreamSynchronize(t->st);
        for (void* p : bufs) cudaFree(p);
    }
};

void op_rows(int rows) { WLK_CHECK(rows >= 1 && rows <= QT_ROUND_ROWS, "rows %d outside [1, %d]", rows, QT_ROUND_ROWS); }

// What the qk-rope and attention kernels index with: slot and position of each row, a layer, the slots' caches.
// `packed`: the rows are laid out as a forward packs them (each slot's rows contiguous, at consecutive positions), which
// the attention tiles assume.
void op_check_rows(wlk_qtext* t, const int32_t* pos, const int32_t* slot, int rows, void* const* kv, int n_slots, int layer,
                   bool packed) {
    op_rows(rows);
    WLK_CHECK(layer >= 0 && layer < t->dims.n_layer, "layer %d outside [0, %d)", layer, t->dims.n_layer);
    WLK_CHECK(n_slots >= 1, "no KV caches");
    std::vector<char> done(n_slots, 0);
    for (int r = 0; r < rows; ++r) {
        WLK_CHECK(slot[r] >= 0 && slot[r] < n_slots, "row %d: slot %d outside [0, %d)", r, slot[r], n_slots);
        WLK_CHECK(kv[slot[r]] != nullptr, "row %d: slot %d has no KV cache", r, slot[r]);
        WLK_CHECK(pos[r] >= 0 && pos[r] < t->dims.max_ctx, "row %d: position %d outside [0, %d)", r, pos[r], t->dims.max_ctx);
        if (!packed) continue;
        if (r > 0 && slot[r] == slot[r - 1]) {
            WLK_CHECK(pos[r] == pos[r - 1] + 1, "row %d: position %d does not follow %d of the same slot", r, pos[r], pos[r - 1]);
        } else {
            WLK_CHECK(!done[slot[r]], "row %d: the rows of slot %d are not contiguous", r, slot[r]);
            done[slot[r]] = 1;
        }
    }
}

void op_rmsnorm(wlk_qtext* t, const float* x, const float* w, void* out, int rows, const int32_t* out_row) {
    WLK_CHECK(x && w && out, "null argument");
    op_rows(rows);
    if (out_row) for (int r = 0; r < rows; ++r) WLK_CHECK(out_row[r] >= -1, "row %d: output row %d", r, out_row[r]);
    OpUpload up{t};
    const int32_t* out_row_d = out_row ? up.put(out_row, rows) : nullptr;
    if (t->act == DT_F32) launch_rmsnorm<float>(t, x, w, out, out_row_d, rows, t->dims.rms_eps);
    else launch_rmsnorm<bf16>(t, x, w, out, out_row_d, rows, t->dims.rms_eps);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

void op_qk_rope(wlk_qtext* t, const float* qkv, const float* qn, const float* kn, const int32_t* pos, const int32_t* slot, int rows,
                void* const* kv, int n_slots, int layer, void* qout) {
    WLK_CHECK(qkv && qn && kn && pos && slot && kv && qout, "null argument");
    op_check_rows(t, pos, slot, rows, kv, n_slots, layer, false);
    OpUpload up{t};
    const int32_t* pos_d = up.put(pos, rows);
    const int32_t* slot_d = up.put(slot, rows);
    void* const* kv_d = up.put(kv, n_slots);
    if (t->act == DT_F32) launch_qk_rope<float>(t, qkv, qn, kn, pos_d, slot_d, kv_d, layer, qout, rows);
    else launch_qk_rope<bf16>(t, qkv, qn, kn, pos_d, slot_d, kv_d, layer, qout, rows);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

void op_attention(wlk_qtext* t, const void* q, const int32_t* pos, const int32_t* slot, int rows, void* const* kv, int n_slots,
                  int layer, void* out) {
    WLK_CHECK(q && pos && slot && kv && out, "null argument");
    op_check_rows(t, pos, slot, rows, kv, n_slots, layer, true);
    std::vector<QTAttnTile> tiles(rows);
    const int n_tiles = make_tiles(pos, slot, rows, tiles.data());
    OpUpload up{t};
    const int32_t* pos_d = up.put(pos, rows);
    const int32_t* slot_d = up.put(slot, rows);
    void* const* kv_d = up.put(kv, n_slots);
    const QTAttnTile* tiles_d = up.put(tiles.data(), n_tiles);
    if (t->act == DT_F32) launch_attention<float>(t, q, pos_d, slot_d, kv_d, tiles_d, n_tiles, layer, out, rows);
    else launch_attention<bf16>(t, q, pos_d, slot_d, kv_d, tiles_d, n_tiles, layer, out, rows);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

void op_swiglu(wlk_qtext* t, const float* gu, void* hid, int rows) {
    WLK_CHECK(gu && hid, "null argument");
    op_rows(rows);
    if (t->act == DT_F32) launch_swiglu<float>(t, gu, hid, rows, t->dims.ffn_dim);
    else launch_swiglu<bf16>(t, gu, hid, rows, t->dims.ffn_dim);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

// The frame adapter over device rows, in chunks of QT_ROUND_ROWS: the residual stream lives in the forward's x workspace.
template <typename T>
void adapt_chunk(wlk_qtext* t, const float* in, int R, int64_t in_ld, float* out, int64_t out_ld) {
    const QTAdapter& A = t->ad;
    const int d = t->dims.d_model, H = A.hidden;
    qt_rows_to_act_kernel<T><<<R, 256, 0, t->st>>>(in, in_ld, (T*)A.a_in, A.in_dim);
    {   GemmArgs g;
        g.A = A.a_in; g.a_type = t->act; g.lda = A.in_dim; g.W = A.Wp; g.w_type = t->act; g.ldw = A.in_dim;
        g.M = R; g.N = d; g.K = A.in_dim;
        g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
        tgemm(t, g); }
    for (int b = 0; b < A.nb; ++b) {
        launch_rmsnorm<T>(t, t->x, A.norm[b], t->xn, nullptr, R, QT_ADAPTER_EPS);
        {   GemmArgs g;
            g.A = t->xn; g.a_type = t->act; g.lda = d; g.W = A.Wgu[b]; g.w_type = t->act; g.ldw = d;
            g.M = R; g.N = 2 * H; g.K = d;
            g.epi.C = A.a_gu; g.epi.c_type = DT_F32; g.epi.ldc = 2 * H;
            tgemm(t, g); }
        launch_swiglu<T>(t, A.a_gu, A.a_hid, R, H);
        {   GemmArgs g;                                 // x + scale * down(...): col_scale, then the residual
            g.A = A.a_hid; g.a_type = t->act; g.lda = H; g.W = A.Wd[b]; g.w_type = t->act; g.ldw = H;
            g.M = R; g.N = d; g.K = H;
            g.epi.col_scale = A.scale; g.epi.scale_cols = d;
            g.epi.residual = t->x; g.epi.ldr = d; g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            tgemm(t, g); }
    }
    CUDA_CHECK(cudaMemcpy2DAsync(out, (size_t)out_ld * 4, t->x, (size_t)d * 4, (size_t)d * 4, R, cudaMemcpyDeviceToDevice, t->st));
    CUDA_CHECK(cudaGetLastError());
}

void adapt(wlk_qtext* t, const float* in, int rows, int64_t in_ld, float* out, int64_t out_ld) {
    WLK_CHECK(t->finalized, "weights not finalized");
    WLK_CHECK(t->has_adapter, "no adapter loaded");
    WLK_CHECK(rows >= 0, "rows %d < 0", rows);
    WLK_CHECK(in_ld >= t->ad.in_dim, "in_ld %lld < in_dim %d", (long long)in_ld, t->ad.in_dim);
    WLK_CHECK(out_ld >= t->dims.d_model, "out_ld %lld < d_model %d", (long long)out_ld, t->dims.d_model);
    WLK_CHECK(rows == 0 || (in && out), "null argument");
    for (int r0 = 0; r0 < rows; r0 += QT_ROUND_ROWS) {
        const int R = std::min(QT_ROUND_ROWS, rows - r0);
        if (t->act == DT_F32) adapt_chunk<float>(t, in + (int64_t)r0 * in_ld, R, in_ld, out + (int64_t)r0 * out_ld, out_ld);
        else adapt_chunk<bf16>(t, in + (int64_t)r0 * in_ld, R, in_ld, out + (int64_t)r0 * out_ld, out_ld);
    }
    CUDA_CHECK(cudaStreamSynchronize(t->st));          // out is complete when the call returns
}

}  // namespace

extern "C" {

int wlk_qtext_create(const wlk_qtext_dims* dims, const wlk_config* cfg, wlk_qtext** out) {
    WLK_API_BEGIN
    create(dims, cfg, out);
    WLK_API_END
}
int wlk_qtext_destroy(wlk_qtext* t) {
    WLK_API_BEGIN
    WLK_CHECK(t != nullptr, "null engine");
    CUDA_CHECK(cudaSetDevice(t->cfg.device));
    destroy(t);
    WLK_API_END
}
int wlk_qtext_load_tensor(wlk_qtext* t, const char* name, const float* host, const int64_t* shape, int ndim) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(name && host && shape && ndim >= 1, "bad arguments");
    load_tensor(t, name, host, shape, ndim);
    WLK_API_END
}
int wlk_qtext_finalize_weights(wlk_qtext* t) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    require_loaded(t->loaded, required(t->dims));
    build_adapter(t);
    t->upload.release();
    t->finalized = true;
    WLK_API_END
}
int wlk_qtext_memory(wlk_qtext* t, size_t* weights, size_t* sessions, size_t* workspace) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    if (weights) *weights = t->bytes_weights;
    if (sessions) *sessions = t->bytes_sessions;
    if (workspace) *workspace = t->bytes_workspace;
    WLK_API_END
}
int wlk_qtext_session_open(wlk_qtext* t, int32_t* sid) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sid, "null out pointer");
    int found = -1;
    for (int i = 0; i < (int)t->sess.size(); ++i) if (!t->sess[i].open) { found = i; break; }
    WLK_CHECK(found >= 0, "all %d sessions in use", (int)t->sess.size());
    QTSession& s = t->sess[found];
    CUDA_CHECK(cudaMalloc(&s.kv, t->kv_bytes));
    t->bytes_sessions += t->kv_bytes;
    s.open = true; s.len = 0;
    *sid = found;
    WLK_API_END
}
int wlk_qtext_session_close(wlk_qtext* t, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    QTSession& s = tsession(t, sid);
    CUDA_CHECK(cudaStreamSynchronize(t->st));
    cudaFree(s.kv);
    t->bytes_sessions -= t->kv_bytes;
    s = QTSession{};
    WLK_API_END
}
int wlk_qtext_session_reset(wlk_qtext* t, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    tsession(t, sid).len = 0;
    WLK_API_END
}
int wlk_qtext_session_len(wlk_qtext* t, int32_t sid, int32_t* len) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(len, "null out pointer");
    *len = tsession(t, sid).len;
    WLK_API_END
}
int wlk_qtext_crop(wlk_qtext* t, int32_t sid, int32_t len) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    QTSession& s = tsession(t, sid);
    WLK_CHECK(len >= 0 && len <= s.len, "crop to %d outside [0, %d]", len, s.len);
    s.len = len;
    WLK_API_END
}
int wlk_qtext_forward(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_offsets,
                      const float* embeds_host, int32_t n_embeds, const int32_t* logit_rows) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sids && row_src && row_offsets && logit_rows && (embeds_host || n_embeds == 0), "null argument");
    forward(t, sids, n, row_src, row_offsets, embeds_host, n_embeds, logit_rows);
    WLK_API_END
}
int wlk_qtext_forward_device(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_offsets,
                             const float* embeds_dev, int64_t embeds_ld, int32_t n_embeds, const int32_t* logit_rows) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sids && row_src && row_offsets && logit_rows && (embeds_dev || n_embeds == 0), "null argument");
    WLK_CHECK(embeds_ld >= t->dims.d_model, "embeds_ld %lld < d_model %d", (long long)embeds_ld, t->dims.d_model);
    forward(t, sids, n, row_src, row_offsets, embeds_dev, n_embeds, logit_rows, embeds_ld);
    WLK_API_END
}
int wlk_qtext_adapt(wlk_qtext* t, const float* in_dev, int32_t rows, int64_t in_ld, float* out_dev, int64_t out_ld) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    adapt(t, in_dev, rows, in_ld, out_dev, out_ld);
    WLK_API_END
}
int wlk_qtext_adapter_dims(wlk_qtext* t, int32_t* in_dim, int32_t* n_blocks, int32_t* hidden) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    if (in_dim) *in_dim = t->has_adapter ? t->ad.in_dim : 0;
    if (n_blocks) *n_blocks = t->ad.nb;
    if (hidden) *hidden = t->ad.hidden;
    WLK_API_END
}
int wlk_qtext_pick(wlk_qtext* t, const int32_t* hist_tokens, int32_t n_hist_tokens, const int32_t* hist_off,
                   const int32_t* hist_len, const int32_t* suppress, int32_t n_suppress, float repetition_penalty,
                   int32_t no_repeat_ngram_size, int32_t max_consecutive, int32_t wait_token_id, int32_t* picks_out,
                   float* value_out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(hist_off && hist_len && picks_out && (hist_tokens || n_hist_tokens == 0) && (suppress || n_suppress == 0), "null argument");
    pick(t, hist_tokens, n_hist_tokens, hist_off, hist_len, suppress, n_suppress, repetition_penalty, no_repeat_ngram_size,
         max_consecutive, wait_token_id, picks_out, value_out);
    WLK_API_END
}
int wlk_qtext_logits(wlk_qtext* t, int32_t row0, int32_t n_rows, float* out_host) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(out_host || n_rows == 0, "null output buffer");
    logits_out(t, row0, n_rows, out_host);
    WLK_API_END
}
int wlk_qtext_op_rmsnorm(wlk_qtext* t, const float* x, const float* w, void* out, int32_t rows, const int32_t* out_row_host) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_rmsnorm(t, x, w, out, rows, out_row_host);
    WLK_API_END
}
int wlk_qtext_op_qk_rope(wlk_qtext* t, const float* qkv, const float* q_norm_w, const float* k_norm_w, const int32_t* row_pos_host,
                         const int32_t* row_slot_host, int32_t rows, void* const* kv_ptrs_host, int32_t n_slots, int32_t layer,
                         void* q_out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_qk_rope(t, qkv, q_norm_w, k_norm_w, row_pos_host, row_slot_host, rows, kv_ptrs_host, n_slots, layer, q_out);
    WLK_API_END
}
int wlk_qtext_op_attention(wlk_qtext* t, const void* q, const int32_t* row_pos_host, const int32_t* row_slot_host, int32_t rows,
                           void* const* kv_ptrs_host, int32_t n_slots, int32_t layer, void* out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_attention(t, q, row_pos_host, row_slot_host, rows, kv_ptrs_host, n_slots, layer, out);
    WLK_API_END
}
int wlk_qtext_op_swiglu(wlk_qtext* t, const float* gu, void* hid, int32_t rows) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_swiglu(t, gu, hid, rows);
    WLK_API_END
}

}  // extern "C"
